"""multi_pose_merge_device / exdet_merge_device on the device, bit for bit: against the reference's own
post_process + merge_outputs stored in tests/golden/detector_tails.npz and against the numpy oracle
(tests/detector_tails_np.py): every row of every class list, stale soft-NMS rows included, NaN / +-inf element for element.
Also the limits (a 4096-row class list is processed, a 4097-row one raises), the radix cut over more than 4096 rows
against np.partition, a non-default stream, untouched inputs and the decoders followed by the tails."""
import numpy as np
import pytest
import torch

from detector_tail_cases import exdet_case, multi_pose_case, oracle_exdet, oracle_multi_pose
from helpers import assert_same_bits, flat_results, golden

pytestmark = pytest.mark.gpu

TAILS = golden("detector_tails")
MP_NAMES = [str(n) for n in TAILS["mp_names"]]
EX_NAMES = [str(n) for n in TAILS["ex_names"]]
NAN_NEG = np.array([0xffc00000], np.uint32).view(np.float32)[0]
NAN_POS = np.array([0x7fc00000], np.uint32).view(np.float32)[0]


@pytest.fixture(scope="module")
def P():
    from centernet_b200 import post_process
    return post_process


def _cuda(arrs):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


@pytest.mark.parametrize("name", EX_NAMES)
def test_exdet_tail_golden(P, name):
    dets, metas, nc, mpi, flip = exdet_case(TAILS, name)
    got = flat_results(P.exdet_merge_device(_cuda(dets), metas, nc, max_per_image=mpi, flip=flip), nc)
    assert_same_bits(got, TAILS[name + "_out"], name)
    if name != "list4096":          # the oracle's Python soft-NMS on a 4096-row list takes minutes
        assert_same_bits(got, flat_results(oracle_exdet(dets, metas, nc, mpi, flip), nc), name + " vs oracle")


@pytest.mark.parametrize("name", MP_NAMES)
def test_multi_pose_tail_golden(P, name):
    dets, metas, nms = multi_pose_case(TAILS, name)
    got = P.multi_pose_merge_device(_cuda(dets), metas, nms=nms)
    assert all(list(r.keys()) == [1] and isinstance(r[1], list) for r in got)
    got = np.array([r[1] for r in got], np.float32)
    assert_same_bits(got, TAILS[name + "_out"], name)
    assert_same_bits(got, oracle_multi_pose(dets, metas, nms), name + " vs oracle")


def _pose(rng, B, K):
    d = np.zeros((B, K, 40), np.float32)
    d[..., 0] = rng.uniform(0, 120, (B, K)); d[..., 1] = rng.uniform(0, 90, (B, K))
    d[..., 2] = d[..., 0] + rng.uniform(2, 30, (B, K)); d[..., 3] = d[..., 1] + rng.uniform(2, 30, (B, K))
    d[..., 4] = np.sort(rng.uniform(0, 1, (B, K)), axis=1)[:, ::-1]
    d[..., 5:39] = rng.uniform(-4, 130, (B, K, 34))
    return d


def _meta(B, h=96, w=128, scale=1.0, seed=0):
    rng = np.random.default_rng(seed)
    return {"c": [np.array([rng.uniform(100, 400), rng.uniform(80, 300)], np.float32) for _ in range(B)],
            "s": [np.float32(512.0) if i % 2 == 0 else np.array([640.0, 384.0], np.float32) for i in range(B)],
            "out_height": h, "out_width": w, "scale": scale}


@pytest.mark.parametrize("nms", [False, True])
def test_multi_pose_k1024(P, nms):
    rng = np.random.default_rng(1024 + nms)
    dets = [_pose(rng, 2, 1024)]
    metas = [_meta(2)]
    got = np.array([r[1] for r in P.multi_pose_merge_device(_cuda(dets), metas, nms=nms)], np.float32)
    assert_same_bits(got, oracle_multi_pose(dets, metas, nms), "K=1024 nms=%s" % nms)


def _exct(rng, n_img, N, nc, classes=None, w=128, h=96):
    d = np.zeros((n_img, N, 14), np.float32)
    d[..., 0] = rng.uniform(-2, w, (n_img, N)); d[..., 1] = rng.uniform(-2, h, (n_img, N))
    d[..., 2] = d[..., 0] + rng.uniform(1, 24, (n_img, N)); d[..., 3] = d[..., 1] + rng.uniform(1, 24, (n_img, N))
    d[..., 4] = rng.uniform(0.01, 1, (n_img, N))
    pool = np.arange(nc) if classes is None else np.asarray(classes)
    d[..., 13] = pool[rng.integers(0, len(pool), (n_img, N))]
    return d


def test_class_list_limit(P):
    """4096 rows of one class are processed (test_exdet_tail_golden[list4096]); 4097 raise after the final copy."""
    rng = np.random.default_rng(4097)
    d = _exct(rng, 2, 4096, 2, classes=(0, 1))
    d[:, :, 13] = 1
    d[1, :, 13] = 0
    d[1, 0, 13] = 1                       # class 1: 4096 + 1 rows over the two halves... of one image
    with pytest.raises(RuntimeError, match="4096"):
        P.exdet_merge_device(_cuda([d]), [_meta(1)], 2, flip=True)


def test_refusals(P):
    rng = np.random.default_rng(5)
    with pytest.raises(ValueError, match="even"):
        P.exdet_merge_device(_cuda([_exct(rng, 1, 7, 3)]), [_meta(1)], 3)
    with pytest.raises(NotImplementedError, match="32768"):
        P.exdet_merge_device(_cuda([_exct(rng, 2, 8194, 3)] * 2), [_meta(1)] * 2, 3, flip=True)
    with pytest.raises(NotImplementedError, match="4096"):
        P.multi_pose_merge_device(_cuda([_pose(rng, 1, 2049)] * 2), [_meta(1)] * 2)
    P.multi_pose_merge_device(_cuda([_pose(rng, 1, 4097)]), [_meta(1)])     # no soft-NMS: no list limit


def _wide_scores(rng, kind, n):
    if kind == "ties":
        return (rng.integers(1, 6, n) / 5).astype(np.float32)
    vals = np.array([0.25, 0.5, 0.0, -0.0, np.inf, -np.inf, NAN_POS, NAN_NEG, -0.25], np.float32)
    p = {"specials": [0.3, 0.3, 0.05, 0.05, 0.05, 0.05, 0.05, 0.1, 0.05],
         "nans": [0.1, 0.1, 0.0, 0.0, 0.05, 0.05, 0.3, 0.4, 0.0]}[kind]
    return vals[rng.choice(len(vals), n, p=p)]


@pytest.mark.parametrize("n,mpi,kind", [(100, 100, "ties"), (4096, 100, "specials"), (4097, 100, "ties"),
                                        (20480, 100, "ties"), (32768, 100, "specials"), (32768, 32767, "ties"),
                                        (9000, 1, "specials"), (5000, 100, "nans"), (30000, 40000, "ties")])
def test_topk_keep_wide_vs_partition(n, mpi, kind):
    """The radix cut against merge_outputs' np.partition threshold: ties at the cut, +-0, +-inf, NaN of both
    signs (the threshold itself NaN in "nans"), and max_per_image above the row count."""
    from centernet_b200._lib import C, ptr, stream_ptr
    rng = np.random.default_rng(n + mpi)
    B, nc, cap = 2, 80, min(n + 3, 32768)      # the image stride may exceed the row count
    rows = np.zeros((B, cap, 5), np.float32)
    rows[:, :n, 4] = _wide_scores(rng, kind, (B, n))
    offs = np.zeros((B, nc + 1), np.int32)
    offs[:, 1:] = n
    offs[1, 1:] = n - 1                        # the second image has one row fewer
    r, o = _cuda([rows, offs])
    keep = torch.full((B, cap), 7, dtype=torch.uint8, device="cuda")
    thr = torch.empty(B, dtype=torch.float32, device="cuda")
    C.topk_keep_wide(ptr(r), B, cap, 5, ptr(o), nc, mpi, ptr(keep), ptr(thr), stream_ptr(r))
    keep, thr = keep.cpu().numpy(), thr.cpu().numpy()
    for i in range(B):
        m = int(offs[i, nc])
        s = rows[i, :m, 4]
        if m > mpi:
            t = np.partition(s, m - mpi)[m - mpi]
            assert_same_bits(thr[i:i + 1], np.array([t], np.float32), "threshold")
            want = s >= t
        else:
            want = np.ones(m, bool)
        np.testing.assert_array_equal(keep[i, :m].astype(bool), want)
        assert (keep[i, m:] == 7).all()


def test_stream_and_inputs_untouched(P):
    dets, metas, nc, mpi, flip = exdet_case(TAILS, "flip_s5")
    src = _cuda(dets)
    before = [t.clone() for t in src]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = P.exdet_merge_device(src, metas, nc, max_per_image=mpi, flip=flip)
    assert_same_bits(flat_results(got, nc), TAILS["flip_s5_out"], "side stream")
    for a, b in zip(src, before):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    dets, metas, nms = multi_pose_case(TAILS, "mp_s5")
    src = _cuda(dets)
    before = [t.clone() for t in src]
    with torch.cuda.stream(s):
        got = P.multi_pose_merge_device(src, metas, nms=nms)
    assert_same_bits(np.array([r[1] for r in got], np.float32), TAILS["mp_s5_out"], "side stream")
    for a, b in zip(src, before):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("agnostic", [False, True])
@pytest.mark.parametrize("flip", [False, True])
def test_exct_decode_then_tail(P, agnostic, flip):
    """exct_decode / agnex_ct_decode followed by the device tail == the decode's .cpu() followed by the oracle."""
    from centernet_b200 import decode as D
    g = torch.Generator().manual_seed(11 + 2 * agnostic + flip)
    scales = (1.0, 1.25)
    B, nc, K, num_dets = 2, 4, 40, 100
    P_ = 2 if flip else 1
    dets, metas = [], []
    for k, sc in enumerate(scales):
        h, w = int(32 * sc), int(40 * sc)
        maps = [torch.sigmoid(torch.randn(P_ * B, 1 if agnostic else nc, h, w, generator=g) * 2 - 2).cuda()
                for _ in range(4)]          # agnostic: one extreme-point map per side, classes from the centre map
        ct = torch.sigmoid(torch.randn(P_ * B, nc, h, w, generator=g) * 2 - 1).cuda()
        fn = D.agnex_ct_decode if agnostic else D.exct_decode
        dets.append(fn(*maps, ct, K=K, num_dets=num_dets))
        metas.append(_meta(B, h=h, w=w, scale=sc, seed=k))
    got = P.exdet_merge_device(dets, metas, nc, max_per_image=100, flip=flip)
    want = oracle_exdet([d.cpu().numpy() for d in dets], metas, nc, 100, flip)
    assert_same_bits(flat_results(got, nc), flat_results(want, nc), "exct end to end")


def test_multi_pose_decode_then_tail(P):
    from centernet_b200 import decode as D
    g = torch.Generator().manual_seed(3)
    B, H, W, K = 2, 48, 64, 100
    dets, metas = [], []
    for k, sc in enumerate((1.0, 0.75)):
        h, w = int(H * sc), int(W * sc)
        heat = torch.sigmoid(torch.randn(B, 1, h, w, generator=g) * 2 - 2).cuda()
        wh = (torch.rand(B, 2, h, w, generator=g) * 20).cuda()
        kps = (torch.randn(B, 34, h, w, generator=g) * 4).cuda()
        dets.append(D.multi_pose_decode(heat, wh, kps, K=K))
        metas.append(_meta(B, h=h, w=w, scale=sc, seed=k))
    got = np.array([r[1] for r in P.multi_pose_merge_device(dets, metas)], np.float32)
    assert_same_bits(got, oracle_multi_pose([d.cpu().numpy() for d in dets], metas, False), "multi_pose end to end")

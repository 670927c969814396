"""CPU: oracle/exct_torch.py, the torch restatement of exct_decode / agnex_ct_decode the GPU tests compare the kernel
with, checked against the numpy oracle (oracle/decode_np.py) on finite maps, against the reference's own outputs
(tests/golden/exct.npz), against its own unchunked form, and its division by 6 against numpy's float32 division.

Bar: every row of every output equal, all 14 columns, the sign of zero included."""
import numpy as np
import pytest
import torch

from helpers import assert_same_bits, golden
from oracle import decode_np as O
from oracle import exct_torch as E


def _maps(B, C, H, W, seed):
    rng = np.random.default_rng(seed)
    maps = [rng.random((B, C, H, W), dtype=np.float32) for _ in range(5)]
    regs = [rng.random((B, 2, H, W)).astype(np.float32) - np.float32(0.5) for _ in range(4)]
    return maps, regs


def _t(*arrs):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)) for a in arrs]


def _agn(maps):
    return [m.max(axis=1, keepdims=True) for m in maps[:4]] + [maps[4]]


@pytest.mark.parametrize("agnostic", [False, True])
@pytest.mark.parametrize("reg", [True, False])
@pytest.mark.parametrize("aggr", [0.0, 0.1])
@pytest.mark.parametrize("B,C,H,W,K,nd", [(2, 3, 12, 16, 7, 300), (1, 2, 9, 11, 13, 1000), (2, 4, 6, 5, 2, 16),
                                          (3, 1, 3, 3, 1, 1), (1, 5, 20, 8, 13, 2048)])
def test_matches_numpy_oracle(B, C, H, W, K, nd, aggr, reg, agnostic):
    maps, regs = _maps(B, C, H, W, 7 * K + C)
    if agnostic:
        maps = _agn(maps)
    if not reg:
        regs = [None] * 4
    f = O.agnex_ct_decode if agnostic else O.exct_decode
    g = E.agnex_ct_decode if agnostic else E.exct_decode
    kw = dict(K=K, num_dets=nd, aggr_weight=aggr)
    want = f(*maps, *regs, **kw)
    got = g(*_t(*maps), *_t(*regs), **kw).numpy()
    if K >= 7:   # tiny K: every tuple may carry a penalty
        assert (want[..., 4] > 0).any()
    assert_same_bits(got, want, "exct_torch vs decode_np")


def test_reproduces_reference_golden():
    """The reference's own outputs (K = 8, num_dets = 60): every row, fillers included."""
    g = golden("exct")
    K, nd = int(g["K"]), int(g["num_dets"])
    maps = _t(g["t"], g["l"], g["b"], g["r"], g["ct"])
    regs = _t(g["t_regr"], g["l_regr"], g["b_regr"], g["r_regr"])
    assert_same_bits(E.exct_decode(*maps, *regs, K=K, num_dets=nd).numpy(), g["dets"], "dets")
    assert_same_bits(E.exct_decode(*maps, K=K, num_dets=nd).numpy(), g["dets_noreg"], "dets_noreg")
    assert_same_bits(E.exct_decode(*maps, *regs, K=K, num_dets=nd, aggr_weight=0.1).numpy(), g["dets_aggr"],
                     "dets_aggr")
    agn = _t(g["t1"], g["l1"], g["b1"], g["r1"], g["ct"])
    assert_same_bits(E.agnex_ct_decode(*agn, *regs, K=K, num_dets=nd).numpy(), g["dets_agn"], "dets_agn")


@pytest.mark.parametrize("agnostic", [False, True])
@pytest.mark.parametrize("kind", ["random", "constant", "nonfinite"])
def test_chunked_equals_unchunked(kind, agnostic):
    """One top index per chunk (many merges of per-chunk tops) against all K^4 tuples sorted at once, on maps where
    most tuples tie and on NaN / inf centre values that must come first."""
    B, C, H, W, K, nd = 2, 3, 10, 12, 9, 700
    maps, regs = _maps(B, C, H, W, 5)
    if kind == "constant":
        maps = [np.full_like(m, 0.5) for m in maps]
    elif kind == "nonfinite":
        ct = maps[4]
        ct[0, 1, 2:5, 3:7] = np.nan
        ct[1, :, 4, :] = np.inf
        ct[1, 2, 6, 2] = -np.inf
    if agnostic:
        maps = _agn(maps)
    g = E.agnex_ct_decode if agnostic else E.exct_decode
    small = g(*_t(*maps), *_t(*regs), K=K, num_dets=nd, chunk_elems=1).numpy()
    whole = g(*_t(*maps), *_t(*regs), K=K, num_dets=nd, chunk_elems=1 << 30).numpy()
    assert_same_bits(small, whole, "chunked vs unchunked")


def test_division_by_six_is_correctly_rounded():
    rng = np.random.default_rng(3)
    x = np.concatenate([rng.standard_normal(200000).astype(np.float32) * np.float32(3),
                        rng.random(100000).astype(np.float32),
                        np.arange(-2000, 2000, dtype=np.float32) / np.float32(7),
                        (rng.random(1000) * 1e-38).astype(np.float32),              # subnormal quotients
                        np.array([0.0, -0.0, 3.4e38, -3.4e38, 1e-45, -1e-45], np.float32)])
    want = x / np.float32(6)
    assert want.dtype == np.float32
    assert_same_bits(E.div6(torch.from_numpy(x)).numpy(), want, "div6 (CPU)")
    if torch.cuda.is_available():
        assert_same_bits(E.div6(torch.from_numpy(x).cuda()).cpu().numpy(), want, "div6 (CUDA)")
    # the trap div6 avoids: a multiplication by fp32(1/6) is off by one ulp somewhere in this sample
    assert not np.array_equal(x * np.float32(1.0 / 6.0), want)


def test_centre_max_follows_torch_max():
    """NaN propagates and takes its class (the first NaN class), ties take the first class, -inf is a number."""
    ct = torch.tensor([[1.0, 3.0, 3.0, 2.0],
                       [1.0, float("nan"), 5.0, float("nan")],
                       [float("-inf"), float("-inf"), float("-inf"), float("-inf")],
                       [float("nan"), 9.0, float("inf"), 0.0],
                       [-0.0, 0.0, -1.0, 0.0]]).T.reshape(1, 4, 1, 5).contiguous()
    v, c = E.centre_max(ct)
    assert c.flatten().tolist() == [1, 1, 0, 0, 0]
    assert np.isnan(v.flatten()[1].item()) and np.isnan(v.flatten()[3].item())
    assert v.flatten()[[0, 2, 4]].tolist() == [3.0, float("-inf"), 0.0]
    assert np.signbit(v.flatten()[4].item())                         # the first class's value, -0 kept
    tv, tc = torch.max(ct, dim=1)
    assert torch.equal(tc, c)

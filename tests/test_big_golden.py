"""North-star geometry (80x128x128, K=100; exct K=40 and K=100) against outputs of the UNMODIFIED reference
(tests/golden/big_*.npz from tests/golden/make_golden_big.py; inputs rebuilt from tests/big_inputs.py and
verified by checksum).  CPU half: pins the numpy oracle.  GPU half: the CUDA path through the C ABI.
Also models/utils.py helpers (A4/A13) and the Reg*Loss gradients (A16) against reference goldens."""
import numpy as np
import pytest
import torch

import big_inputs as BI
from helpers import assert_dets_bits, assert_dets_equal, golden
from oracle import decode_np as O

TOL = 1e-4


def dev(*arrs):
    return [None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrs]


def _ctdet(kind):
    g = golden("big_ctdet_" + kind)
    heat, wh, reg = BI.ctdet_inputs(kind)
    assert BI.checksum(heat, wh, reg) == g["crc"], "seeded inputs differ from the ones the golden was made with"
    return g, heat, wh, reg


def _multi_pose():
    g = golden("big_multi_pose")
    ins = BI.multi_pose_inputs()
    assert BI.checksum(*ins) == g["crc"]
    return g, ins


def _exct():
    g = golden("big_exct")
    maps, regs = BI.exct_inputs()
    assert BI.checksum(*maps, *regs) == g["crc"]
    return g, maps, regs


# --------------------------------------------------------------------------- CPU: the oracle
@pytest.mark.parametrize("kind", ["noise", "blobs"])
def test_oracle_ctdet_big(kind):
    g, heat, wh, reg = _ctdet(kind)
    np.testing.assert_array_equal(O.ctdet_decode(heat, wh, reg, K=100), g["dets"])
    np.testing.assert_array_equal(O.ctdet_decode(heat, wh, None, K=100), g["dets_noreg"])


def test_oracle_multi_pose_big():
    g, (heat, wh, kps, reg, hm_hp, hp_off) = _multi_pose()
    np.testing.assert_array_equal(O.multi_pose_decode(heat, wh, kps, reg, hm_hp, hp_off, K=100), g["dets"])


@pytest.mark.parametrize("K,aggr,key", [(40, 0.0, "dets_k40"), (40, 0.1, "dets_k40_aggr"), (100, 0.0, "dets_k100")])
def test_oracle_exct_big(K, aggr, key):
    g, maps, regs = _exct()
    got = O.exct_decode(*maps, *regs, K=K, num_dets=1000, aggr_weight=aggr)
    assert (g[key][..., 4] > 0).sum() > 0
    assert_dets_equal(g[key], got, positive_only=True, what=key)


def test_oracle_agnex_big():
    g, maps, regs = _exct()
    t1, l1, b1, r1 = [m.max(axis=1, keepdims=True) for m in maps[:4]]
    got = O.agnex_ct_decode(t1, l1, b1, r1, maps[4], *regs, K=40, num_dets=1000)
    assert_dets_equal(g["dets_agn_k40"], got, positive_only=True, what="agnex_k40")


def test_oracle_utils():
    g = golden("utils")
    np.testing.assert_array_equal(O.transpose_and_gather_feat(g["feat"], g["ind"]), g["tg"])
    np.testing.assert_array_equal(O.gather_feat(g["feat3"], g["ind3"]), g["g"])


# --------------------------------------------------------------------------- GPU: the CUDA path
@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["noise", "blobs"])
def test_gpu_ctdet_big(kind):
    from centernet_b200 import decode as D
    g, heat, wh, reg = _ctdet(kind)
    h, w_, r = dev(heat, wh, reg)
    assert_dets_equal(g["dets"], D.ctdet_decode(h, w_, reg=r, K=100).cpu().numpy(), atol=TOL, what="big ctdet")
    assert_dets_equal(g["dets_noreg"], D.ctdet_decode(h, w_, K=100).cpu().numpy(), atol=TOL, what="big ctdet noreg")
    # batch 1 (the reference's actual inference mode, src/test.py:60-62) and the host-buffer entry
    assert_dets_equal(g["dets"][:1], D.ctdet_decode(h[:1], w_[:1], reg=r[:1], K=100).cpu().numpy(), atol=TOL,
                      what="big ctdet B=1")
    got = D.ctdet_decode_from_host(torch.from_numpy(heat), torch.from_numpy(wh), reg=torch.from_numpy(reg), K=100)
    assert_dets_equal(g["dets"], got.numpy(), atol=TOL, what="big ctdet from host")


@pytest.mark.gpu
def test_gpu_multi_pose_big():
    from centernet_b200 import decode as D
    g, ins = _multi_pose()
    heat, wh, kps, reg, hm_hp, hp_off = dev(*ins)
    got = D.multi_pose_decode(heat, wh, kps, reg=reg, hm_hp=hm_hp, hp_offset=hp_off, K=100).cpu().numpy()
    assert_dets_bits(g["dets"], got, what="big multi_pose")


@pytest.mark.gpu
@pytest.mark.parametrize("K,aggr,key", [(40, 0.0, "dets_k40"), (40, 0.1, "dets_k40_aggr"), (100, 0.0, "dets_k100")])
def test_gpu_exct_big(K, aggr, key):
    from centernet_b200 import decode as D
    g, maps, regs = _exct()
    got = D.exct_decode(*dev(*maps), *dev(*regs), K=K, num_dets=1000, aggr_weight=aggr).cpu().numpy()
    assert_dets_equal(g[key], got, atol=TOL, positive_only=True, what=key)


@pytest.mark.gpu
def test_gpu_exct_k100_aggr_vs_oracle():
    """What detectors/exdet.py:39-51 passes (K=100) with aggr_weight 0.1; EVERY row against the oracle
    (which shares the kernel's tie rule), including the non-positive fillers."""
    from centernet_b200 import decode as D
    _, maps, regs = _exct()
    want = O.exct_decode(*maps, *regs, K=100, num_dets=1000, aggr_weight=0.1)
    got = D.exct_decode(*dev(*maps), *dev(*regs), K=100, num_dets=1000, aggr_weight=0.1).cpu().numpy()
    np.testing.assert_array_equal(got[..., 4], want[..., 4])
    np.testing.assert_array_equal(got[..., 13], want[..., 13])
    np.testing.assert_allclose(got, want, rtol=0, atol=TOL)


@pytest.mark.gpu
def test_gpu_agnex_big():
    from centernet_b200 import decode as D
    g, maps, regs = _exct()
    t1, l1, b1, r1 = [m.max(axis=1, keepdims=True) for m in maps[:4]]
    got = D.agnex_ct_decode(*dev(t1, l1, b1, r1, maps[4]), *dev(*regs), K=40, num_dets=1000).cpu().numpy()
    assert_dets_equal(g["dets_agn_k40"], got, atol=TOL, positive_only=True, what="agnex_k40")


@pytest.mark.gpu
def test_gpu_utils_golden():
    """A4/A13: models/utils.py mirrors against the reference's outputs, and the gather is differentiable."""
    from centernet_b200 import utils as U
    g = golden("utils")
    feat, ind, feat3, ind3, hm17, logits = dev(g["feat"], g["ind"], g["feat3"], g["ind3"], g["hm17"], g["logits"])
    np.testing.assert_array_equal(U._transpose_and_gather_feat(feat, ind).cpu().numpy(), g["tg"])
    np.testing.assert_array_equal(U._gather_feat(feat3, ind3).cpu().numpy(), g["g"])
    np.testing.assert_array_equal(U.flip_tensor(feat).cpu().numpy(), g["flip_tensor"])
    fi = [list(map(int, e)) for e in g["flip_idx"]]
    np.testing.assert_array_equal(U.flip_lr(hm17, fi).cpu().numpy(), g["flip_lr"])
    np.testing.assert_array_equal(U.flip_lr_off(feat, fi).cpu().numpy(), g["flip_lr_off"])
    np.testing.assert_allclose(U._sigmoid(logits.clone()).cpu().numpy(), g["sigmoid"], rtol=0, atol=1e-6)
    # gradient of the gather == autograd of the reference formulation (permute + gather), incl. repeated indices
    ind_rep = ind.clone(); ind_rep[:, 1] = ind_rep[:, 0]
    f1 = feat.clone().requires_grad_(True)
    go = torch.randn(2, 9, 34, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    (U._transpose_and_gather_feat(f1, ind_rep) * go).sum().backward()
    f2 = feat.clone().requires_grad_(True)
    ref = f2.permute(0, 2, 3, 1).contiguous().view(2, -1, 34).gather(1, ind_rep.unsqueeze(2).expand(2, 9, 34))
    (ref * go).sum().backward()
    assert torch.allclose(f1.grad, f2.grad, rtol=0, atol=1e-6)


@pytest.mark.gpu
def test_gpu_reference_losses_train_through_overlay_gather():
    """ADVICE r1 (high): the reference's own loss classes call _transpose_and_gather_feat; with the overlay the
    regression heads must still receive gradient."""
    from centernet_b200 import utils as U
    g = golden("losses"); gg = golden("losses_grads")
    output, ind, mask, target = dev(g["output"], g["ind"], g["mask"], g["target"])
    o = output.clone().requires_grad_(True)
    pred = U._transpose_and_gather_feat(o, ind)                     # models/losses.py:139-149 (RegL1Loss.forward)
    m = mask.unsqueeze(2).expand_as(pred).float()
    loss = torch.nn.functional.l1_loss(pred * m, target * m, reduction="sum") / (m.sum() + 1e-4)
    loss.backward()
    np.testing.assert_allclose(float(loss), float(g["reg_l1"]), rtol=1e-5)
    np.testing.assert_allclose(o.grad.cpu().numpy(), gg["reg_l1_grad"], rtol=0, atol=1e-6)


@pytest.mark.gpu
def test_gpu_reg_loss_gradients_golden():
    """A16: gradients of all four Reg losses against the reference's autograd (losses_grads.npz)."""
    from centernet_b200 import losses as L
    g = golden("losses"); gg = golden("losses_grads")
    output, ind, mask, target, wmask = dev(g["output"], g["ind"], g["mask"], g["target"], g["wmask"])
    for name, crit, args in (("reg_l1", L.RegL1Loss(), (mask, ind, target)),
                             ("reg_sl1", L.RegLoss(), (mask, ind, target)),
                             ("norm_l1", L.NormRegL1Loss(), (mask, ind, target.abs() + 0.5)),
                             ("weighted_l1", L.RegWeightedL1Loss(), (wmask, ind, target))):
        o = output.clone().requires_grad_(True)
        loss = crit(o, *args)
        loss.backward()
        np.testing.assert_allclose(float(loss), float(g[name]), rtol=1e-5, err_msg=name)
        np.testing.assert_allclose(o.grad.cpu().numpy(), gg[name + "_grad"], rtol=1e-5, atol=1e-6, err_msg=name)

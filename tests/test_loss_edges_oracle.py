"""CPU checks of the references tests/test_loss_edges_gpu.py uses: the numpy splat oracle and the fp64
restatements of the focal and Reg*Loss formulas against tests/golden/loss_edges.npz (the reference's own
functions), so that a GPU failure points at the kernel and not at its yardstick."""
import hashlib

import numpy as np
import pytest

from helpers import assert_same_bits, golden
from oracle import image_np
from test_loss_edges_gpu import assert_close_class, focal_ref64, reg_ref64, splat_ref

G = golden("loss_edges")


def test_gaussian2d_digests():
    """oracle/image_np.gaussian2d, cast to fp32, is the reference's gaussian2D bit for bit at r = 0 .. 200."""
    dig = G["gauss_digest"]
    for r in range(dig.shape[0]):
        d = 2 * r + 1
        h = image_np.gaussian2d(d, d / 6).astype(np.float32)
        assert hashlib.sha256(h.tobytes()).digest() == dig[r].tobytes(), r


@pytest.mark.parametrize("name", [str(n) for n in G["splat_names"]])
def test_splat_oracle(name):
    k = lambda s: G["s_%s_%s" % (name, s)]
    C, H, W = (int(v) for v in k("chw"))
    assert_same_bits(splat_ref(k("cls"), k("cx"), k("cy"), k("rad"), k("valid"), C, H, W), k("hm"), name)


@pytest.mark.parametrize("name", [str(n) for n in G["focal_names"]])
def test_focal_ref64(name):
    x, gt, logits = G["f_%s_x" % name], G["f_%s_gt" % name], bool(G["f_%s_logits" % name])
    loss, grad = focal_ref64(x, gt, logits)
    want_l, want_g = G["f_%s_loss" % name], G["f_%s_grad" % name]
    if name == "logit_extremes":
        # fp64 and fp32 clamp at different points: 1e-4 vs 1e-4f; only the non-finite pattern is comparable here
        assert_close_class([loss], [want_l], None, 0, name)
        assert_close_class(grad, want_g, None, 0, name)
        return
    assert_close_class([loss], [want_l], 1e-5, 0, name + " loss")
    assert_close_class(grad, want_g, 1e-4, 1e-6, name + " grad")


@pytest.mark.parametrize("name", [str(n) for n in G["reg_names"]])
def test_reg_ref64(name):
    k = lambda s: G["r_%s_%s" % (name, s)]
    loss, grad = reg_ref64(int(k("mode")), k("output"), k("mask"), k("ind"), k("target"))
    np.testing.assert_allclose(loss, k("loss"), rtol=1e-5)
    np.testing.assert_allclose(grad, k("grad"), rtol=1e-5, atol=1e-6)

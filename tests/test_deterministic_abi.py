"""CPU: the C ABI of deterministic mode.  Every call here fails validation or only queries sizes, so nothing reaches a
GPU: the workspace query grows with the switch and keeps its default-mode values, the fp32-only configurations are
refused in deterministic mode, and a channels-last grad_input is no longer refused there."""
import pytest

SHAPES = [
    (16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1),      # dla_34 64@128^2 -> 64
    (16, 256, 256, 32, 32, 3, 3, 1, 1, 1, 1),
    (2, 64, 272, 12, 12, 3, 3, 1, 1, 1, 1),       # Cout > 256: the weight pass's fp32 kernel needs partials
    (2, 12, 11, 5, 9, 3, 3, 2, 1, 1, 2),          # ragged, strided, grouped
    (33, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1),     # two batch chunks
]


@pytest.fixture
def C():
    from centernet_b200 import _C
    _C.dcnv2_set_deterministic(0)
    yield _C
    _C.dcnv2_set_deterministic(0)


def test_workspace_query_grows_in_deterministic_mode(C):
    q = C.dcnv2_backward_workspace_bytes
    base = [q(*s) for s in SHAPES]
    assert all(v > 0 for v in base)
    C.dcnv2_set_deterministic(1)
    det = [q(*s) for s in SHAPES]
    C.dcnv2_set_deterministic(0)
    assert [q(*s) for s in SHAPES] == base            # default mode: unchanged by the switch having been on
    for s, b, d in zip(SHAPES, base, det):
        assert d >= b and d % 16 == 0, s
    # 64@128^2: the fixed-point dX of one batch chunk (32 images x 16384 positions x 64 channels x 8 bytes) on top
    assert det[0] - base[0] >= 16 * 128 * 128 * 64 * 8
    assert det[4] - base[4] >= 32 * 128 * 128 * 64 * 8
    # what the tensor-core backward does not cover stays 0 in both modes
    C.dcnv2_set_deterministic(1)
    assert q(2, 64, 64, 32, 32, 5, 5, 1, 2, 1, 1) == 0
    assert q(1, 32, 32, 8192, 8192, 3, 3, 1, 1, 1, 1) == 0


def test_fp32_only_configurations_refused(C):
    """Deterministic mode: no workspace, or anisotropic stride, is CNB_EUNSUPPORTED (before any CUDA call)."""
    fake = 1 << 20       # never dereferenced: validation fails first
    args = dict(b=2, cin=64, h=8, w=8, cout=64)
    C.dcnv2_set_deterministic(1)
    with pytest.raises(RuntimeError, match="deterministic mode"):
        C.dcnv2_backward(fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, args["b"], args["cin"], args["h"],
                         args["w"], args["cout"], 3, 3, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0)
    wsb = C.dcnv2_backward_workspace_bytes(2, 64, 64, 8, 8, 3, 3, 1, 1, 1, 1)
    with pytest.raises(RuntimeError, match="deterministic mode"):
        C.dcnv2_backward(fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 2, 64, 8, 8, 64, 3, 3,
                         2, 1, 1, 1, 1, 1, 1, fake, wsb, 0)
    # a default-mode-sized workspace is too small in deterministic mode
    C.dcnv2_set_deterministic(0)
    small = C.dcnv2_backward_workspace_bytes(2, 64, 64, 8, 8, 3, 3, 1, 1, 1, 1)
    C.dcnv2_set_deterministic(1)
    assert small < wsb
    with pytest.raises(RuntimeError, match="deterministic mode"):
        C.dcnv2_backward(fake, fake, fake, fake, fake, fake, fake, fake, fake, fake, 2, 64, 8, 8, 64, 3, 3,
                         1, 1, 1, 1, 1, 1, 1, fake, small, 0)


def test_channels_last_grad_input_accepted(C):
    """cnb_dcnv2_backward_ex in deterministic mode: with the deterministic-mode workspace a channels-last grad_input
    passes the mode's checks; the call below stops only at the layout rule that holds in both modes (cin / dg a
    multiple of 32), never at a deterministic-mode refusal."""
    fake = 1 << 20
    C.dcnv2_set_deterministic(1)
    wsb = C.dcnv2_backward_workspace_bytes(2, 48, 64, 8, 8, 3, 3, 1, 1, 1, 1)
    with pytest.raises(RuntimeError) as e:
        C.dcnv2_backward_ex(fake, 1, fake, fake, fake, fake, fake, 1, fake, fake, fake, fake, 2, 48, 8, 8, 64, 3, 3, 1, 1,
                            1, 1, fake, wsb, 0)
    assert "multiple of 32" in str(e.value) and "deterministic" not in str(e.value)
    C.dcnv2_set_deterministic(0)


def test_focal_workspace_holds_the_partials(C):
    # one (pos, neg) double pair per CTA of the loss kernels behind the accumulator block
    assert C.focal_workspace_bytes(32 * 80 * 128 * 128) >= 256 + 16 * 5120

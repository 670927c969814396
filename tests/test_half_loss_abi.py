"""The C ABI of the bf16 / fp16 loss calls, as far as it can be checked without a GPU: the symbols are bound, a dtype
code is validated before anything else (no CUDA call is reached: every pointer here is NULL), the calls that have
no fp32 form say so, and the workspace query is the one the fp32 losses use."""
import pytest

from centernet_b200._lib import _C

F32, BF16, F16 = 0, 1, 2

# name -> arguments with the dtype code at index `at` (pointers 0, sizes 1)
CALLS = {
    "focal_loss_ex": ([0, F32, 0, 1, 0, 0, 0, 0, 0], 1),
    "focal_grad_ex": ([0, F32, 0, 1, 0, 0, 0, 0, 0], 1),
    "focal_splat_loss_ex": ([0, F32, 0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0], 1),
    "focal_splat_grad_ex": ([0, 1, 0, 0, F32, 0], 4),
    "reg_loss_ex": ([0, F32, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0], 1),
    "reg_loss_grad_ex": ([0, F32, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, 0, 0], 1),
    "gather_feat_ex": ([0, F32, 0, 0, 1, 1, 1, 1, 0], 1),
    "gather_feat_backward_ex": ([0, 0, 0, F32, 1, 1, 1, 1, 0], 3),
}


def call(name, code):
    args, at = CALLS[name]
    args = list(args)
    args[at] = code
    return getattr(_C, name)(*args)


@pytest.mark.parametrize("name", sorted(CALLS))
def test_symbol_is_bound(name):
    assert callable(getattr(_C, name))


@pytest.mark.parametrize("code", [3, -1])
@pytest.mark.parametrize("name", sorted(CALLS))
def test_unknown_dtype_code_is_refused_first(name, code):
    with pytest.raises(RuntimeError, match="unknown dtype code %d" % code):
        call(name, code)


@pytest.mark.parametrize("code", [BF16, F16])
@pytest.mark.parametrize("name", sorted(CALLS))
def test_null_pointers_are_refused_before_any_launch(name, code):
    with pytest.raises(RuntimeError, match="cnb_%s: null pointer" % name):
        call(name, code)


@pytest.mark.parametrize("name", ["focal_grad_ex", "focal_splat_grad_ex", "reg_loss_ex", "reg_loss_grad_ex"])
def test_calls_without_an_fp32_form_say_so(name):
    with pytest.raises(NotImplementedError, match="bf16 / fp16 only"):
        call(name, F32)


@pytest.mark.parametrize("name,fp32", [("focal_loss_ex", "cnb_focal_loss"), ("focal_splat_loss_ex", "cnb_focal_splat_loss"),
                                       ("gather_feat_ex", "cnb_gather_feat")])
def test_fp32_code_is_the_fp32_call(name, fp32):
    """The fp32 code forwards to the fp32 entry point: its own argument check answers."""
    with pytest.raises(RuntimeError, match="%s: null pointer" % fp32):
        call(name, F32)


def test_splat_list_length_limit_is_kept():
    args = list(CALLS["focal_splat_loss_ex"][0])
    args[0] = args[2] = args[3] = args[4] = args[5] = args[6] = args[13] = args[15] = 16   # non-NULL, never read
    args[1], args[8] = BF16, 129
    with pytest.raises(NotImplementedError, match="at most 128 objects"):
        _C.focal_splat_loss_ex(*args)


def test_workspace_query_is_unchanged():
    for n in (1, 4099, 64 * 80 * 128 * 128):
        assert _C.focal_workspace_bytes(n) == 256 + 16384 * 16

"""CPU: the C-ABI library loads and exports every symbol include/centernet_b200.h declares and _C binds
each of them with the header's parameters; argument validation works without a GPU (no compute calls here)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    """{name: [parameter declarations]} of every function the header declares ((void) is no parameter)."""
    src = open(os.path.join(ROOT, "include", "centernet_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return {name: [p.strip() for p in params.split(",") if p.strip() != "void"]
            for name, params in re.findall(r"\b(cnb_[a-z0-9_]+)\s*\(([^)]*)\)", src)}


def test_every_declared_symbol_is_exported():
    lib = ctypes.CDLL(os.path.join(ROOT, "centernet_b200", "lib", "libcenternet_b200.so"))
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), "missing export " + n
    lib.cnb_version.restype = ctypes.c_int
    assert lib.cnb_version() >= 100


def test_every_declared_function_is_bound_with_its_parameters():
    """_C binds exactly the header's functions, each positionally with the header's parameters in order: a float
    where the header has float or double, an int for a pointer or an integer type.  Reads __doc__ only; a call with
    made-up pointers could reach the GPU."""
    from centernet_b200._lib import _C   # the extension itself; centernet_b200._C is its device-guarding proxy
    decls = _declared()
    bound = {n for n in dir(_C) if not n.startswith("_") and callable(getattr(_C, n))}
    assert bound == {n[4:] for n in decls}
    for name, params in decls.items():
        if name in ("cnb_last_error", "cnb_select_plan_info"):   # bound by hand: return a str / a dict
            continue
        want = ["float" if "*" not in p and re.search(r"\b(float|double)\b", p) else "int" for p in params]
        sig = getattr(_C, name[4:]).__doc__.splitlines()[0]
        got = [(int(i), "float" if "float" in t.lower() else "int" if "int" in t.lower() else t)
               for i, t in re.findall(r"\barg(\d+): ([\w. |]+)", sig)]
        assert got == list(enumerate(want)), "%s: header (%s), bound %s" % (name, ", ".join(params), sig)


def test_pybind_layer_and_validation():
    from centernet_b200 import _C
    assert _C.version() >= 100
    assert _C.topk_workspace_bytes(64, 80, 128, 128, 100) > 0
    # bad arguments are rejected before any CUDA call (status EINVAL -> RuntimeError)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.ctdet_decode(0, 0, 0, 0, 1, 80, 128, 128, 100, 0, 0, 0, 0)
    with pytest.raises(RuntimeError, match="exceeds"):
        _C.topk(16, 1, 1, 4, 4, 17, 0, 0, 0, 0, 0, 0, 16, 1 << 20, 0)
    assert "exceeds" in _C.last_error()


def test_select_plan_info():
    """cnb_select_plan_info: the selection's plan without a launch (no GPU needed: without a device the plan is
    made for 132 SMs)."""
    from centernet_b200 import _C
    keys = ["hot", "n_cta", "wb", "max_slots", "seg_cap", "fused_finalize", "use_tma", "rb", "local_img"]
    p = _C.select_plan_info(256, 64, 80, 128, 128, 100, 1, 4)
    assert sorted(p) == sorted(keys)
    assert p["hot"] == 1 and p["use_tma"] == 1 and p["rb"] == 128 and p["fused_finalize"] == 1
    assert p["seg_cap"] == 256 and p["wb"] == 4 and 1 <= p["n_cta"] <= 192 and p["max_slots"] >= 2
    assert _C.select_plan_info(256, 64, 80, 128, 128, 200, 1, 4)["seg_cap"] == 200
    assert _C.select_plan_info(256, 64, 80, 128, 128, 100, 1, 2)["hot"] == 1          # fp16 / bf16 map
    assert _C.select_plan_info(258, 64, 80, 128, 128, 100, 1, 2)["use_tma"] == 0      # misaligned: generic path
    assert _C.select_plan_info(256, 64, 80, 128, 128, 100, 0, 4)["hot"] == 0          # no peak test
    big = _C.select_plan_info(256, 1, 80, 128, 128, 1000, 1, 4)
    assert big["hot"] == 0 and big["fused_finalize"] == 0 and big["max_slots"] * 1000 <= 8192
    one = _C.select_plan_info(256, 1, 3, 128, 128, 100, 1, 4)
    assert one["n_cta"] == 1 and one["local_img"] == 1
    assert _C.select_plan_info(256, 100, 1, 128, 128, 100, 1, 4)["local_img"] == 1    # C=1: one plane per image
    strips = _C.select_plan_info(256, 2, 4, 200, 152, 64, 1, 4)
    assert strips["hot"] == 0 and strips["rb"] < 200
    with pytest.raises(NotImplementedError):
        _C.select_plan_info(256, 1, 80, 128, 128, 1025, 1, 4)
    with pytest.raises(RuntimeError, match="exceeds"):
        _C.select_plan_info(256, 1, 1, 4, 4, 17, 1, 4)
    with pytest.raises(RuntimeError, match="elem_size"):
        _C.select_plan_info(256, 1, 1, 4, 4, 1, 1, 8)


def test_no_cpu_fallback():
    import torch
    from centernet_b200 import decode
    with pytest.raises(NotImplementedError):
        decode.ctdet_decode(torch.rand(1, 2, 8, 8), torch.rand(1, 2, 8, 8))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "centernet_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cpp")):
                txt = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "oracle/" not in txt and "oracle." not in txt, f


def test_validation_of_later_entry_points():
    """Argument checks of the logits decode, DCNv2 workspace, PSROI pooling and edge aggregation run before any
    CUDA call, so they can be exercised without a GPU."""
    from centernet_b200 import _C
    # fused-sigmoid decode: same workspace as the heat-map path in the hot geometry (no heat map is materialised),
    # plus one map for other geometries
    hot = _C.ctdet_logits_workspace_bytes(0, 64, 80, 128, 128, 100)
    assert 0 < hot <= _C.topk_workspace_bytes(64, 80, 128, 128, 100)
    generic = _C.ctdet_logits_workspace_bytes(0, 2, 5, 40, 60, 33)
    assert generic >= 2 * 5 * 40 * 60 * 4
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.ctdet_decode_logits(0, 0, 0, 0, 1, 80, 128, 128, 100, 0, 0, 0, 0)
    # DCNv2 tensor-core forward: re-tiled weights (hi + lo, 18 chunks of [64][32]) + channels-last copy of the input
    ws = _C.dcnv2_workspace_bytes(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)
    assert ws == 18 * 2 * 64 * 32 * 4 + 16 * 128 * 128 * 64 * 4
    assert _C.dcnv2_workspace_bytes(16, 64, 64, 128, 128, 5, 5, 1, 2, 1, 1) == 0      # 25 taps: fp32 path only
    # PSROI pooling: position-sensitive channels must exist
    with pytest.raises(RuntimeError, match="channels"):
        _C.psroi_pooling_forward(16, 16, 0, 16, 16, 1, 8, 9, 9, 2, 2, 1, 0.25, 4, 2, 3, 3, 2, 0.0, 0)
    with pytest.raises(RuntimeError, match="offsets"):
        _C.psroi_pooling_forward(16, 16, 0, 16, 16, 1, 8, 9, 9, 2, 3, 0, 0.25, 2, 2, 3, 3, 2, 0.0, 0)
    with pytest.raises(RuntimeError, match="in-place"):
        _C.edge_aggregate(16, 16, 1, 1, 8, 8, 0.1, 1, 0)


def test_dcnv2_backward_workspace_query_and_switches():
    """cnb_dcnv2_backward_workspace_bytes: positive for what the tensor-core backward covers, 0 where the fp32 kernels must
    run (more than 9 taps, bad shapes, images beyond the 32-bit in-image indexing); the deterministic switch is a
    process-wide flag; cnb_dcnv2_backward_ex validates before any CUDA call."""
    from centernet_b200 import _C
    q = _C.dcnv2_backward_workspace_bytes
    base = q(16, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1)
    assert base > 0 and base % 16 == 0
    assert q(32, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) > base            # grows with the batch ...
    # ... but the column gradient (671 MB per 16 images here) is held to ~1.5 GiB: at B=256 the workspace is the two
    # channels-last copies (2 x 1.07 GB) + max(gy tiles + dcol chunk, the weight pass's 2.1 GB of dY tiles), not 10.7 GB of dcol
    assert q(256, 64, 64, 128, 128, 3, 3, 1, 1, 1, 1) < 6 * (1 << 30)
    assert q(2, 64, 64, 32, 32, 5, 5, 1, 2, 1, 1) == 0                  # 25 taps
    assert q(2, 64, 64, 32, 32, 3, 3, 1, 1, 1, 3) == 0                  # cin not divisible by the groups
    assert q(1, 32, 32, 8192, 8192, 3, 3, 1, 1, 1, 1) == 0              # image too large for 32-bit in-image offsets
    assert q(2, 12, 5, 9, 11, 3, 3, 2, 1, 1, 2) > 0                     # ragged, strided, grouped: covered
    # an empty output grid (2x2 image, 3x3 kernel, no padding) is rejected by every call, so every fp32 query returns 0
    for det in (0, 1):
        _C.dcnv2_set_deterministic(det)
        for query in (q, _C.dcnv2_workspace_bytes, _C.dcnv2_prepared_workspace_bytes):
            assert query(2, 64, 64, 2, 2, 3, 3, 1, 0, 1, 1) == 0
    _C.dcnv2_set_deterministic(0)
    assert _C.dcnv2_get_deterministic() == 0
    _C.dcnv2_set_deterministic(1)
    assert _C.dcnv2_get_deterministic() == 1
    _C.dcnv2_set_deterministic(0)
    with pytest.raises(RuntimeError, match="null pointer"):
        _C.dcnv2_backward_ex(0, 1, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 2, 64, 8, 8, 64, 3, 3, 1, 1, 1, 1, 0, 0, 0)

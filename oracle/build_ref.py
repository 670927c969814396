"""Recipe for oracle/_ref (TEST INFRASTRUCTURE): the reference DCNv2 on the GPU.

Compiles the reference's two THC-free kernel files UNMODIFIED, from where they lie under
/root/reference, for sm_90a, together with oracle/ref_host.cu (the cuBLAS restatement of the
removed-THC host loop, dcn_v2_cuda.c:61-97,161-231,243-330) into

    oracle/_ref/libdcnv2_ref.so

No reference source is copied into the repository: only the built library lands in oracle/_ref/
(git-ignored, NOT gpurun-ignored, so it travels to the GPU box like our own .so files).  On the
GPU box /root/reference does not exist; build() then only reports whether the prebuilt library
is there.  Run: ``python -m oracle.build_ref [--force]``.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
LIB = os.path.join(OUT, "libdcnv2_ref.so")
REF_CUDA = "/root/reference/src/lib/models/networks/DCNv2/src/cuda"
REF_SOURCES = [os.path.join(REF_CUDA, "dcn_v2_im2col_cuda.cu"),
               os.path.join(REF_CUDA, "dcn_v2_psroi_pooling_cuda.cu")]
HOST = os.path.join(HERE, "ref_host.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def available():
    return os.path.exists(LIB)


def build(force=False):
    """Returns the library path, or None when neither the reference sources nor a prebuilt
    library are present (never raises for a missing reference: the checker is optional)."""
    have_src = all(os.path.exists(s) for s in REF_SOURCES)
    if not have_src:
        return LIB if available() else None
    srcs = REF_SOURCES + [HOST]
    if not force and available() and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return LIB
    os.makedirs(OUT, exist_ok=True)
    cmd = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-shared", "-Xcompiler", "-fPIC",
           "-cudart", "static", "-I" + REF_CUDA] + srcs + ["-lcublas", "-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return LIB


# ---------------------------------------------------------------- the reference's Cython soft-NMS (N2 oracle pin)
REF_NMS = "/root/reference/src/lib/external/nms.pyx"


def nms_lib_path():
    import sysconfig
    return os.path.join(OUT, "nms" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def build_nms(force=False):
    """oracle/_ref/nms<ext>.so = the reference's src/lib/external/nms.pyx (soft_nms :77-169, soft_nms_39 :171-275)
    through cython + gcc.  The file is compiled as it lies except for ONE declaration outside those functions:
    `np.int_t` (the hard-NMS helper `nms`, :32) no longer exists in NumPy 2 and is retyped `np.intp_t` in a
    temporary copy that is deleted after the build (nothing of the reference enters the repository)."""
    import shutil
    import sysconfig
    import tempfile
    lib = nms_lib_path()
    if not os.path.exists(REF_NMS):
        return lib if os.path.exists(lib) else None
    if not force and os.path.exists(lib) and os.path.getmtime(lib) >= os.path.getmtime(REF_NMS):
        return lib
    import numpy
    os.makedirs(OUT, exist_ok=True)
    tmp = tempfile.mkdtemp(prefix="cnb_nms_")
    try:
        src = open(REF_NMS).read().replace("np.int_t", "np.intp_t")
        with open(os.path.join(tmp, "nms.pyx"), "w") as f:
            f.write(src)
        for cmd in (["cython", "-3", os.path.join(tmp, "nms.pyx"), "-o", os.path.join(tmp, "nms.c")],
                    ["gcc", "-O2", "-shared", "-fPIC", "-Wno-cpp", "-Wno-unused-function", "-I" + numpy.get_include(),
                     "-I" + sysconfig.get_paths()["include"], os.path.join(tmp, "nms.c"), "-o", lib]):
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("oracle/_ref nms build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    return lib


def load_nms():
    """The compiled reference module (or None when it was never built)."""
    import importlib.util
    path = build_nms()
    if path is None or not os.path.exists(path):
        return None
    spec = importlib.util.spec_from_file_location("nms", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
    print(build_nms(force="--force" in sys.argv))

"""Recipe for oracle/_ref/libdcnv2_ref_f64.so (TEST INFRASTRUCTURE): the reference's float64 DCNv2 build
(_ext.dcn_v2_double, build_double.py) on the GPU.

Compiles the reference's two float64 kernel files UNMODIFIED, from where they lie under /root/reference, for
sm_90a, together with oracle/ref_host_f64.cu (the cuBLAS DGEMM / DGEMV restatement of the THC host loop of
dcn_v2_cuda_double.c).  It is a library of its own: the float and the double files export the same extern "C"
launcher names (modulated_deformable_im2col_cuda, DeformablePSROIPoolForward, ...), so they cannot share
libdcnv2_ref.so.  No reference source is copied into the repository; only the built library lands in oracle/_ref/
(git-ignored, and shipped with the tree to the GPU machine like our own .so files).  Where /root/reference does
not exist, build() only reports whether the prebuilt library is there.
Run: ``python -m oracle.build_ref_f64 [--force]``.
"""
import os
import subprocess
import sys

from .build_ref import NVCC, OUT, REF_CUDA

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(OUT, "libdcnv2_ref_f64.so")
REF_SOURCES = [os.path.join(REF_CUDA, "dcn_v2_im2col_cuda_double.cu"),
               os.path.join(REF_CUDA, "dcn_v2_psroi_pooling_cuda_double.cu")]
HOST = os.path.join(HERE, "ref_host_f64.cu")


def available():
    return os.path.exists(LIB)


def build(force=False):
    """Returns the library path, or None when neither the reference sources nor a prebuilt library are present."""
    if not all(os.path.exists(s) for s in REF_SOURCES):
        return LIB if available() else None
    srcs = REF_SOURCES + [HOST]
    if not force and available() and all(os.path.getmtime(s) <= os.path.getmtime(LIB) for s in srcs):
        return LIB
    os.makedirs(OUT, exist_ok=True)
    # dcn_v2_psroi_pooling_cuda_double.cu launches 1024-thread blocks; compiled for sm_90a its kernels need more than
    # 64 registers a thread, and the launch then fails with "too many resources requested" (which the file only
    # prints).  That file alone is compiled with the registers capped at 64 -- a compiler flag, the source stays as
    # it is -- so its kernels run; the DCNv2 kernels keep the compiler's choice.
    base = [NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-Xcompiler", "-fPIC", "-I" + REF_CUDA]
    psroi_obj = os.path.join(OUT, "dcn_v2_psroi_pooling_cuda_double.o")
    r = subprocess.run(base + ["-maxrregcount=64", "-c", REF_SOURCES[1], "-o", psroi_obj], capture_output=True,
                       text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref f64 build failed: %s\n%s" % (r.stdout, r.stderr))
    cmd = base + ["-shared", "-cudart", "static", REF_SOURCES[0], HOST, psroi_obj, "-lcublas", "-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("oracle/_ref f64 build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))

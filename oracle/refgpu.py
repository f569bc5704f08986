"""TEST / MEASUREMENT INFRASTRUCTURE — ctypes binding of oracle/_ref/libblitzar_ref_gpu.so: the
reference's own bucket-method GPU kernels (unmodified sources compiled for sm_90a by
oracle/ref_build/Makefile, driver oracle/ref_build/ref_gpu_driver.cu). Used only by tests/ to put
the reference's KERNELS beside ours on the same GPU; the product never imports this module."""
import ctypes as C
import os
import warnings

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libblitzar_ref_gpu.so")
_lib = None


def available():
    """The library is built by the current recipe (it has ref_gpu_probe) and its kernels can run on
    the current device. A library that is present but unusable is reported, not silently ignored."""
    if not os.path.exists(LIB_PATH):
        return False
    if not hasattr(_load(), "ref_gpu_probe"):
        why = "was built by an older recipe (no ref_gpu_probe)"
    else:
        rc = _load().ref_gpu_probe()
        if rc == 0:
            return True
        if rc != 209:  # cudaErrorNoKernelImageForDevice
            warnings.warn(f"{LIB_PATH}: no usable CUDA device (CUDA error {rc}); treating the "
                          "reference GPU kernels as unavailable.", stacklevel=2)
            return False
        why = "has no kernel image for this device"
    warnings.warn(f"{LIB_PATH} {why}; rebuild it (build() with BLITZAR_REFERENCE set). "
                  "Treating the reference GPU kernels as unavailable.", stacklevel=2)
    return False


def _load():
    global _lib
    if _lib is None:
        _lib = C.CDLL(LIB_PATH)
    return _lib


def bucket_msm(generators, scalars):
    """generators uint8 [n,160] (sxt_ristretto255), scalars uint8 [n,32] -> (element_p3 bytes
    [1,160], whole-call ms incl. H2D/D2H, kernels-only ms)."""
    n = len(scalars)
    assert generators.shape == (n, 160) and scalars.shape == (n, 32)
    generators, scalars = np.ascontiguousarray(generators), np.ascontiguousarray(scalars)
    out = np.zeros((1, 160), dtype=np.uint8)
    times = (C.c_float * 2)()
    rc = _load().ref_gpu_bucket_msm(C.c_void_p(out.ctypes.data), C.c_void_p(generators.ctypes.data),
                                 C.c_void_p(scalars.ctypes.data), C.c_uint(n), times)
    if rc != 0:
        raise RuntimeError("reference GPU kernels failed")
    return out, times[0], times[1]

"""The reference's own hog.c with channels and bilinear orientations (oracle/ref_vl_hog_channels.cpp), built into oracle/_ref.

TEST INFRASTRUCTURE ONLY.  Importable from tests/ and bench_vl_hog.py -- never from the product package.  build() compiles the
wrapper against the reference tree ($REF, default /root/reference) with the flags of oracle/Makefile (-O2 -ffp-contract=off:
baseline x86-64 without FMA, as the reference's CMake builds it); without the reference tree it keeps a library built before.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ref_vl_hog_channels.cpp")
_PATH = os.path.join(_HERE, "_ref", "libref_vl_hog_channels.so")
_lib = None


def build() -> None:
    ref = os.environ.get("REF", "/root/reference")
    hog_c = os.path.join(ref, "include", "rcr", "hog.c")
    if not os.path.isfile(hog_c):
        return
    if os.path.exists(_PATH) and os.path.getmtime(_PATH) >= max(os.path.getmtime(_SRC), os.path.getmtime(hog_c)):
        return
    os.makedirs(os.path.dirname(_PATH), exist_ok=True)
    subprocess.run(["g++", "-O2", "-fPIC", "-ffp-contract=off", "-std=c++14", "-shared", "-I", os.path.dirname(hog_c), "-o", _PATH,
                    _SRC, "-lm"], check=True)


def available() -> bool:
    return os.path.exists(_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libref_vl_hog_channels.so is not built")
        _lib = C.CDLL(_PATH)
    return _lib


def vl_hog(image: np.ndarray, cell_size: int, num_bins: int, variant: int = 1, bilinear: bool = False) -> np.ndarray:
    """vl_hog_put_image + vl_hog_extract of one float image, (h, w) or planar (channels, h, w), with the bilinear switch set.
    Returns the planar [dd, hogH, hogW]."""
    image = np.ascontiguousarray(image, dtype=np.float32)
    if image.ndim == 2:
        image = image[None]
    c, h, w = image.shape
    fp = image.ctypes.data_as(C.POINTER(C.c_float))
    dims = (C.c_int * 3)()
    if lib().ref_vl_hog_channels(variant, num_bins, fp, w, h, c, cell_size, int(bool(bilinear)), None, dims):
        raise RuntimeError("vl_hog_new failed")
    out = np.zeros((dims[2], dims[1], dims[0]), dtype=np.float32)
    lib().ref_vl_hog_channels(variant, num_bins, fp, w, h, c, cell_size, int(bool(bilinear)),
                              out.ctypes.data_as(C.POINTER(C.c_float)), dims)
    return out

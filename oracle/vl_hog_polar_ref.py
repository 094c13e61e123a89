"""The reference's own hog.c through vl_hog_put_polar_field (oracle/ref_vl_hog_polar.cpp), built into oracle/_ref.

TEST INFRASTRUCTURE ONLY.  Importable from tests/ and bench_vl_hog_polar.py -- never from the product package.  build()
compiles the wrapper against the reference tree ($REF, default /root/reference) with the flags of oracle/Makefile (-O2
-ffp-contract=off: baseline x86-64 without FMA, as the reference's CMake builds it); without the reference tree it keeps a
library built before.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ref_vl_hog_polar.cpp")
_PATH = os.path.join(_HERE, "_ref", "libref_vl_hog_polar.so")
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
            raise RuntimeError("oracle/_ref/libref_vl_hog_polar.so is not built")
        _lib = C.CDLL(_PATH)
    return _lib


def vl_hog_polar(modulus: np.ndarray, angle: np.ndarray, cell_size: int, num_bins: int, variant: int = 1, directed: bool = True,
                 bilinear: bool = False) -> np.ndarray:
    """vl_hog_put_polar_field + vl_hog_extract of one (h, w) gradient field, modulus and angle, with the bilinear switch set.
    Returns the planar [dd, hogH, hogW]."""
    modulus = np.ascontiguousarray(modulus, dtype=np.float32)
    angle = np.ascontiguousarray(angle, dtype=np.float32)
    if modulus.ndim != 2 or modulus.shape != angle.shape:
        raise ValueError("modulus and angle must be (h, w) fields of one shape")
    h, w = modulus.shape
    mp, ap = modulus.ctypes.data_as(C.POINTER(C.c_float)), angle.ctypes.data_as(C.POINTER(C.c_float))
    dims = (C.c_int * 3)()
    args = (variant, num_bins, mp, ap, w, h, int(bool(directed)), cell_size, int(bool(bilinear)))
    if lib().ref_vl_hog_polar(*args, None, dims):
        raise RuntimeError("vl_hog_new failed")
    out = np.zeros((dims[2], dims[1], dims[0]), dtype=np.float32)
    lib().ref_vl_hog_polar(*args, out.ctypes.data_as(C.POINTER(C.c_float)), dims)
    return out

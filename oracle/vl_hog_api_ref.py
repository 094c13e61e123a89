"""The reference's own hog.c through its VlHog object (oracle/ref_vl_hog_api.cpp), and the hog.h driver program
(oracle/vl_hog_driver.cpp) compiled against the reference's hog.h, both built into oracle/_ref.

TEST INFRASTRUCTURE ONLY.  Importable from tests/ and bench_vl_hog_api.py -- never from the product package.  build()
compiles both against the reference tree ($REF, default /root/reference) with the flags of oracle/Makefile (-O2
-ffp-contract=off: baseline x86-64 without FMA, as the reference's CMake builds it); without the reference tree it keeps what
was built before.  The driver binary needs nothing but libc and libstdc++ at run time.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ref_vl_hog_api.cpp")
_DRIVER_SRC = os.path.join(_HERE, "vl_hog_driver.cpp")
_PATH = os.path.join(_HERE, "_ref", "libref_vl_hog_api.so")
DRIVER = os.path.join(_HERE, "_ref", "vl_hog_driver_ref")
GLYPH = 21
_lib = None


def _fresh(target: str, deps) -> bool:
    return os.path.exists(target) and os.path.getmtime(target) >= max(os.path.getmtime(d) for d in deps)


def build() -> None:
    ref = os.environ.get("REF", "/root/reference")
    hog_c = os.path.join(ref, "include", "rcr", "hog.c")
    if not os.path.isfile(hog_c):
        return
    os.makedirs(os.path.dirname(_PATH), exist_ok=True)
    flags = ["g++", "-O2", "-ffp-contract=off", "-std=c++14"]
    if not _fresh(_PATH, [_SRC, hog_c]):
        subprocess.run(flags + ["-fPIC", "-shared", "-I", os.path.dirname(hog_c), "-o", _PATH, _SRC, "-lm"], check=True)
    if not _fresh(DRIVER, [_DRIVER_SRC, hog_c]):
        subprocess.run(flags + ["-I", os.path.join(ref, "include"), "-o", DRIVER, _DRIVER_SRC, "-lm", "-lpthread"], check=True)


def available() -> bool:
    return os.path.exists(_PATH)


def lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError("oracle/_ref/libref_vl_hog_api.so is not built")
        l = C.CDLL(_PATH)
        l.ref_hog_new.restype = C.c_void_p
        l.ref_hog_new.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
        for name in ("ref_hog_delete", "ref_hog_put_image", "ref_hog_put_polar", "ref_hog_dims", "ref_hog_extract", "ref_hog_render",
                     "ref_hog_permutation", "ref_hog_glyphs"):
            getattr(l, name).restype = None
        l.ref_hog_delete.argtypes = [C.c_void_p]
        l.ref_hog_put_image.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        l.ref_hog_put_polar.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        l.ref_hog_dims.argtypes = [C.c_void_p, C.c_void_p]
        l.ref_hog_extract.argtypes = [C.c_void_p, C.c_void_p]
        l.ref_hog_render.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
        l.ref_hog_permutation.argtypes = [C.c_void_p, C.c_void_p]
        l.ref_hog_glyphs.argtypes = [C.c_void_p, C.c_void_p]
        _lib = l
    return _lib


class Hog:
    """One VlHog of the reference: vl_hog_new(variant, num_bins, transposed) with the bilinear switch set."""

    def __init__(self, variant: int, num_bins: int, transposed: bool = False, bilinear: bool = False):
        self.num_bins = num_bins
        self.h = lib().ref_hog_new(int(variant), int(num_bins), int(bool(transposed)), int(bool(bilinear)))

    def __del__(self):
        try:
            if self.h:
                lib().ref_hog_delete(self.h)
                self.h = None
        except Exception:   # interpreter shutdown
            pass

    def dims(self):
        """(hogW, hogH, dd, glyph size) of the last put."""
        d = (C.c_int * 4)()
        lib().ref_hog_dims(self.h, d)
        return tuple(d)

    def _extract(self) -> np.ndarray:
        w, h, dd, _ = self.dims()
        out = np.zeros((dd, h, w), np.float32)
        lib().ref_hog_extract(self.h, out.ctypes.data)
        return out

    def put_image(self, image: np.ndarray, cell_size: int) -> np.ndarray:
        """vl_hog_put_image + vl_hog_extract of a (C, H, W) or (H, W) float32 buffer read as width W, height H (x fastest);
        returns [dd][hogH][hogW] in the buffer's coordinates."""
        a = np.ascontiguousarray(image, np.float32)
        c, h, w = (1,) + a.shape if a.ndim == 2 else a.shape
        lib().ref_hog_put_image(self.h, a.ctypes.data, w, h, c, int(cell_size))
        return self._extract()

    def put_polar(self, modulus: np.ndarray, angle: np.ndarray, cell_size: int, directed: bool = True) -> np.ndarray:
        m, a = np.ascontiguousarray(modulus, np.float32), np.ascontiguousarray(angle, np.float32)
        h, w = m.shape
        lib().ref_hog_put_polar(self.h, m.ctypes.data, a.ctypes.data, int(bool(directed)), w, h, int(cell_size))
        return self._extract()

    def render(self, features: np.ndarray, image: np.ndarray = None) -> np.ndarray:
        """vl_hog_render of [dd][h][w] features into image (h * 21, w * 21), zeros when None; returns the image."""
        f = np.ascontiguousarray(features, np.float32)
        _, h, w = f.shape
        img = np.zeros((h * GLYPH, w * GLYPH), np.float32) if image is None else np.array(image, np.float32, copy=True, order="C")
        lib().ref_hog_render(self.h, img.ctypes.data, f.ctypes.data, w, h)
        return img

    def permutation(self) -> np.ndarray:
        dd = self.dims()[2]
        out = np.zeros(dd, np.int64)
        lib().ref_hog_permutation(self.h, out.ctypes.data)
        return out

    def glyphs(self) -> np.ndarray:
        out = np.zeros((self.num_bins, GLYPH, GLYPH), np.float32)
        lib().ref_hog_glyphs(self.h, out.ctypes.data)
        return out

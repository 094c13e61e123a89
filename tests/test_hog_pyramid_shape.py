"""The HOG pyramid's level rule on the host (sd_hog_pyramid_shape), its refusals, and the resize oracle the GPU pyramid tests pin
the levels to.

A level of a W x H frame at scale s is floor(W s + 0.5) x floor(H s + 0.5) px (double arithmetic), and its cells are those of the
dense HOG of that level; a level below 4 px or with an empty cell grid is empty (hog_w = hog_h = 0).  oracle.resize_linear_u8
must equal cv2.resize(INTER_LINEAR) at every level size used here, so that it is a valid pin for the device's resize."""
import ctypes as C
import math

import numpy as np
import pytest


@pytest.fixture(scope="module")
def lib():
    from superviseddescent_b200 import build, _capi
    build.build()
    return _capi.lib()


def _shape(lib, w, h, s, cs, K, variant):
    o = [C.c_int(-7) for _ in range(5)]
    rc = lib.sd_hog_pyramid_shape(w, h, s, cs, K, variant, *[C.byref(v) for v in o])
    return rc, tuple(v.value for v in o)


def _expected(w, h, s, cs, K, variant):
    lw, lh = int(math.floor(w * s + 0.5)), int(math.floor(h * s + 0.5))
    hw, hh = (lw + cs // 2) // cs, (lh + cs // 2) // cs
    dd = 3 * K + 4 if variant == 1 else 4 * K
    if lw < 4 or lh < 4 or hw <= 0 or hh <= 0:
        hw = hh = 0
    return lw, lh, hw, hh, dd


def _scales():
    return [2.0 ** (-l / 5) for l in range(-5, 25)] + [0.5, 1.0, 1.5, 2.0, 4.0, 0.01, 1e-9, 0.3333333333333333, 2.5]


def test_level_rule_matches_restatement(lib):
    rng = np.random.default_rng(5)
    sizes = [(1280, 720), (640, 480), (333, 211), (97, 131), (4, 4), (3, 50), (1, 1)] + \
            [tuple(int(v) for v in rng.integers(1, 2000, 2)) for _ in range(40)]
    n = 0
    for w, h in sizes:
        for s in _scales():
            for cs, K, variant in [(8, 9, 1), (4, 4, 0), (11, 16, 1), (32, 1, 0), (1, 7, 1)]:
                rc, got = _shape(lib, w, h, s, cs, K, variant)
                assert rc == 0 and got == _expected(w, h, s, cs, K, variant), (w, h, s, cs, K, variant, got)
                n += 1
    assert n > 5000


def test_scale_one_and_half(lib):
    assert _shape(lib, 1280, 720, 1.0, 8, 9, 1) == (0, (1280, 720, 160, 90, 31))
    assert _shape(lib, 1280, 720, 0.5, 8, 9, 1) == (0, (640, 360, 80, 45, 31))
    assert _shape(lib, 333, 211, 0.5, 8, 9, 1)[1][:2] == (167, 106)        # 166.5 + 0.5 rounds up
    assert _shape(lib, 7, 7, 0.5, 4, 9, 1) == (0, (4, 4, 1, 1, 31))
    assert _shape(lib, 7, 7, 0.4, 4, 9, 1) == (0, (3, 3, 0, 0, 31))         # below 4 px: empty
    assert _shape(lib, 100, 100, 0.04, 8, 9, 1) == (0, (4, 4, 1, 1, 31))    # (4 + 4) // 8: one cell
    assert _shape(lib, 100, 100, 0.04, 9, 9, 1) == (0, (4, 4, 0, 0, 31))    # 4 px but no cell of 9: empty


@pytest.mark.parametrize("args", [
    (640, 480, 0.0, 8, 9, 1), (640, 480, -0.5, 8, 9, 1), (640, 480, 4.000001, 8, 9, 1), (640, 480, float("nan"), 8, 9, 1),
    (640, 480, float("inf"), 8, 9, 1), (640, 480, 1.0, 0, 9, 1), (640, 480, 1.0, 33, 9, 1), (640, 480, 1.0, 8, 0, 1),
    (640, 480, 1.0, 8, 17, 1), (640, 480, 1.0, 8, 9, 2), (0, 480, 1.0, 8, 9, 1), (640, -1, 1.0, 8, 9, 1),
    (2 ** 30, 480, 1.0, 8, 9, 1)])
def test_refusals(lib, args):
    rc, got = _shape(lib, *args)
    assert rc == 1 and got == (-7,) * 5


def test_null_outputs_refused(lib):
    v = C.c_int()
    assert lib.sd_hog_pyramid_shape(64, 64, 1.0, 8, 9, 1, None, C.byref(v), C.byref(v), C.byref(v), C.byref(v)) == 1


def test_pyramid_call_refusals_without_work(lib):
    """sd_hog_pyramid refuses a null context before anything else (the rest of its refusals run on the GPU)."""
    s = (C.c_double * 1)(1.0)
    assert lib.sd_hog_pyramid(None, None, s, 1, 8, 9, 1, None, None) == 1
    assert lib.sd_hog_correlate(None, None, 9, 1, None, 1, 6, 6, None, 0, 0, None) == 1


def test_oracle_resize_equals_cv2_at_level_sizes(oracle):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    bad = total = 0
    for W, H in [(1280, 720), (333, 211), (97, 131)]:
        img = cv2.GaussianBlur(rng.integers(0, 256, (H, W), dtype=np.uint8), (0, 0), 2)
        for s in _scales()[:30] + [0.5, 1.5]:
            w, h = int(math.floor(W * s + 0.5)), int(math.floor(H * s + 0.5))
            if w < 4 or h < 4:
                continue
            a = oracle.resize_linear_u8(img, w, h)
            b = cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
            bad += int((a != b).sum())
            total += a.size
    assert total > 10_000_000 and bad == 0

"""CPU checks of the sample-warp rule and its helpers: sample_warp_ref.window equals the same window of cv2.warpAffine's whole V
bit for bit over rotations (0, 90 and 180 degrees included), scales 0.25 to 4, reflections, shear and anisotropic scale, V smaller
and larger than the frame, and windows across V's and the frame's edges; rotation_warp, invert_warp and warp_landmarks against
cv2 and each other."""
import numpy as np
import pytest

import sample_warp_ref as SW
from superviseddescent_b200 import api as sd

cv2 = pytest.importorskip("cv2")


def _frame(h, w, seed):
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 256, (h, w), dtype=np.uint8)
    return cv2.GaussianBlur(g, (5, 5), 1.5)


def _warps():
    c = (61.5, 40.25)
    out = [(sd.rotation_warp(c, a, s), size) for a in (0, 90, 180, -90, 17.5, -44.0, 133.0) for s in (0.25, 1.0, 4.0)
           for size in ((120, 80), (37, 23), (301, 190))]
    out += [(np.array([[-1.0, 0, 119], [0, 1, 0]]), (120, 80)),                 # the mirror at the frame's size
            (np.array([[1.0, 0, 0], [0, -1, 79]]), (120, 80)),                  # upside down
            (np.array([[0.7, 0.45, -10.3], [-0.2, 1.6, 5.7]]), (150, 60)),       # shear, anisotropic scale
            (np.array([[2.5, 0.0, 3.1], [0.0, 0.4, -7.9]]), (90, 200)),
            (np.array([[-0.8, 0.3, 130.2], [0.5, 0.9, -20.0]]), (140, 110))]      # reflection with rotation
    return out


def test_window_equals_cv2_window_of_whole_V():
    g = _frame(80, 120, 3)
    rng = np.random.default_rng(5)
    n = 0
    for M, size in _warps():
        V = SW.materialise(g, M, size)
        for _ in range(6):
            P = int(rng.integers(1, 40)) * 2
            x0, y0 = int(rng.integers(-P - 4, size[0] + 4)), int(rng.integers(-P - 4, size[1] + 4))
            got = SW.window(g, M, size, x0, y0, P)
            assert got is not None
            assert np.array_equal(got, SW.crop(V, x0, y0, P)), (M, size, x0, y0, P)
            n += 1
        # the whole of V as one window
        whole = SW.window(g, M, size, 0, 0, max(size))
        assert np.array_equal(whole[:size[1], :size[0]], V)
    assert n > 300


def test_invalid_warps_are_refused():
    g = _frame(40, 50, 1)
    assert SW.window(g, np.array([[np.nan, 0, 0], [0, 1, 0]]), (10, 10), 0, 0, 4) is None
    assert SW.window(g, np.eye(2, 3), (0, 10), 0, 0, 4) is None
    assert SW.window(g, np.array([[1e9, 0, 0], [0, 1, 0]]), (10, 10), 0, 0, 4) is None


def test_rotation_warp_is_the_inverse_of_get_rotation_matrix():
    for c in ((0.0, 0.0), (320.5, 240.25), (-17.0, 1e3)):
        for a in (0, 15, 30, 45, 60, 90, 180, -33.3, 270, 721.0):
            for s in (0.25, 1.0, 1.7, 4.0):
                want = cv2.invertAffineTransform(cv2.getRotationMatrix2D(c, a, s))
                assert np.max(np.abs(sd.rotation_warp(c, a, s) - want)) <= 1e-12, (c, a, s)


def test_invert_and_warp_landmarks_round_trip():
    rng = np.random.default_rng(2)
    M = rng.normal(size=(7, 2, 3)) * [[1, 1, 50], [1, 1, 50]]
    Mi = sd.invert_warp(M)
    eye = np.einsum("nij,njk->nik", np.concatenate([M[:, :, :2]], 0), Mi[:, :, :2])
    assert np.allclose(eye, np.eye(2), atol=1e-12)
    assert np.allclose(sd.invert_warp(Mi), M, atol=1e-9)
    x = rng.uniform(0, 300, (7, 44)).astype(np.float32)
    back = sd.warp_landmarks(sd.warp_landmarks(x, Mi), M)
    assert back.dtype == np.float32 and np.allclose(back, x, atol=1e-3)
    one = sd.warp_landmarks(x[0], M[0])
    assert one.shape == (44,) and np.array_equal(one, sd.warp_landmarks(x[:1], M[0])[0])
    # x' = m0 x + m1 y + m2 in float64
    L = 22
    want = M[0, 0, 0] * x[0, :L].astype(np.float64) + M[0, 0, 1] * x[0, L:].astype(np.float64) + M[0, 0, 2]
    assert np.array_equal(one[:L], want.astype(np.float32))


def test_helpers_refuse_malformed_shapes():
    with pytest.raises(ValueError):
        sd.invert_warp(np.zeros((3, 3)))
    with pytest.raises(ValueError):
        sd.invert_warp(np.zeros((2, 3)))                 # singular
    with pytest.raises(ValueError):
        sd.warp_landmarks(np.zeros((2, 44), np.float32), np.zeros((3, 2, 3)))
    with pytest.raises(ValueError):
        sd.warp_landmarks(np.zeros((2, 44), np.float32), np.zeros((2, 2)))
    with pytest.raises(ValueError):
        sd._warp_table(np.zeros((2, 3, 3)), None, np.zeros((2, 2)), "cpu")
    with pytest.raises(ValueError):
        sd._warp_table(np.zeros((2, 2, 3)), np.zeros((3, 2)), None, "cpu")

"""The face chip rule of tests/face_chip_ref.py on the CPU: the warp equals cv2.warpAffine(INTER_LINEAR | WARP_INVERSE_MAP,
BORDER_CONSTANT, 0) bit for bit for 8-bit frames of 1, 3 and 4 channels and float frames of 1 and 3, for chips inside the frame,
past each edge, wholly outside it and on the frame's own grid, at scales 0.25 to 4 and rotations over the full circle; the fit
equals numpy's least squares; align_mean landmarks fit without rotation at the box's scale; and invalid faces are refused."""
import numpy as np
import pytest

import face_chip_ref as ref
import synth

cv2 = pytest.importorskip("cv2")


def _frame(C, dtype, seed, H=71, W=97):
    rng = np.random.default_rng(seed)
    g = np.stack([synth.smooth_images(1, H, W, seed=seed + c, sigma=1.0)[0] for c in range(C)], axis=-1)
    g = g ^ rng.integers(0, 8, g.shape, dtype=np.uint8)           # texture, so every tap weight shows
    g = g[:, :, 0] if C == 1 else g
    return (g.astype(np.float32) / np.float32(255) * np.float32(1.7)) if dtype == np.float32 else g


def _cv2(frame, M, w, h):
    out = cv2.warpAffine(frame, M, (int(w), int(h)), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                         borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    return out.reshape(h, w, -1)


def _similarity(scale, angle, tx, ty):
    a, b = scale * np.cos(angle), scale * np.sin(angle)
    return np.array([[a, -b, tx], [b, a, ty]])


def _cases(H, W, rng):
    """(M, w, h): inside, past each edge, wholly outside, the identity, and random scales, rotations and chip sizes."""
    out = [(_similarity(1.0, 0.0, 0.0, 0.0), W, H),                      # exactly the frame's grid: a copy
           (_similarity(1.0, 0.0, 5.0, 3.0), 30, 20),                    # an integer shift
           (_similarity(0.7, 0.3, W / 3, H / 4), 40, 40),                # inside
           (_similarity(1.2, 0.1, -25.0, H / 3), 40, 30),                # past the left edge
           (_similarity(1.2, -0.1, W - 20.0, H / 3), 40, 30),            # past the right edge
           (_similarity(0.9, 0.2, W / 4, -20.0), 30, 40),                # past the top
           (_similarity(0.9, -0.2, W / 4, H - 15.0), 30, 40),            # past the bottom
           (_similarity(1.0, 0.5, -500.0, -400.0), 25, 25),              # wholly outside
           (_similarity(2.0, np.pi, W + 10.0, H + 10.0), 21, 13)]        # rotated half a turn, from past the far corner
    for _ in range(24):
        s, t = 2.0 ** rng.uniform(-2, 2), rng.uniform(-np.pi, np.pi)
        w, h = (int(v) for v in rng.integers(3, 64, 2))
        out.append((_similarity(s, t, rng.uniform(-30, W + 30), rng.uniform(-30, H + 30)), w, h))
    return out


@pytest.mark.parametrize("C,dtype", [(1, np.uint8), (3, np.uint8), (4, np.uint8), (1, np.float32), (3, np.float32)])
def test_warp_equals_cv2(C, dtype):
    rng = np.random.default_rng(C * 7 + (dtype == np.float32))
    frame = _frame(C, dtype, seed=C)
    H, W = frame.shape[:2]
    for M, w, h in _cases(H, W, rng):
        got = ref.warp(frame, M, w, h)
        want = _cv2(frame, M, w, h)
        assert got.shape == want.shape and got.dtype == want.dtype
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (M, w, h)


def test_float_warp_keeps_nan_and_inf_taps():
    """Every tap is read and multiplied: an inf beside a weight-0 tap gives NaN, as in cv2."""
    frame = _frame(1, np.float32, seed=3)
    frame[20, 30], frame[40, 50] = np.inf, np.nan
    for M, w, h in [(_similarity(1.0, 0.0, 10.25, 5.0), 40, 40), (_similarity(0.8, 0.4, 12.0, 2.0), 50, 50)]:
        got, want = ref.warp(frame, M, w, h), _cv2(frame, M, w, h)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fit_equals_lstsq():
    rng = np.random.default_rng(5)
    for _ in range(200):
        L = int(rng.integers(2, 30))
        n = int(rng.integers(2, L + 1))
        idx = rng.permutation(L)[:n]
        u = rng.uniform(0, 200, (n, 2))
        x = rng.uniform(-100, 900, 2 * L).astype(np.float32)
        a, b, tx, ty = ref.fit(x, idx, u)
        # [px; py] = [[ux, -uy, 1, 0], [uy, ux, 0, 1]] [a, b, tx, ty]
        A = np.zeros((2 * n, 4))
        A[:n, 0], A[:n, 1], A[:n, 2] = u[:, 0], -u[:, 1], 1
        A[n:, 0], A[n:, 1], A[n:, 3] = u[:, 1], u[:, 0], 1
        rhs = np.concatenate([x[idx], x[L + idx]]).astype(np.float64)
        want = np.linalg.lstsq(A, rhs, rcond=None)[0]
        got = np.array([a, b, tx, ty])
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want))), (got, want)
        M, Mi = ref.matrices(a, b, tx, ty)
        back = np.vstack([Mi, [0, 0, 1]]) @ np.vstack([M, [0, 0, 1]])
        assert np.allclose(back, np.eye(3), rtol=0, atol=1e-12 * max(1.0, abs(tx), abs(ty)))


def test_align_mean_landmarks_fit_the_box(golden):
    """Landmarks exactly align_mean(mean, box) of a square box fit the default template without rotation (|b| within float
    rounding of the landmarks) at the box's scale: a = box side (1 + 2 padding) / chip side."""
    mean = golden.mean68.astype(np.float32).ravel()
    L = mean.size // 2
    size, padding = 112, 0.25
    tm = ref.template(mean, size, size, padding)
    for x0, y0, s in [(100, 50, 80), (-20, 300, 200), (640, 360, 37)]:
        x = np.concatenate([(mean[:L] + np.float32(0.5)) * np.float32(s) + np.float32(x0),
                            (mean[L:] + np.float32(0.5)) * np.float32(s) + np.float32(y0)]).astype(np.float32)
        a, b, tx, ty = ref.fit(x, np.arange(L), tm)
        scale = s * (1 + 2 * padding) / size
        assert abs(b) <= 1e-6 * scale and abs(a - scale) <= 1e-6 * scale
        # the box's corner (x0, y0) lands on the padding border of the chip
        M, _ = ref.matrices(a, b, tx, ty)
        corner = M @ np.array([padding / (1 + 2 * padding) * size] * 2 + [1.0])
        assert np.allclose(corner, [x0, y0], atol=1e-3 * s)


def test_invalid_faces():
    frame = _frame(3, np.uint8, seed=9)
    L = 5
    idx = np.arange(L)
    u = np.array([[10.0, 10], [30, 10], [20, 20], [12, 30], [28, 30]])
    good = np.concatenate([u[:, 0] * 1.5 + 20, u[:, 1] * 1.5 + 10]).astype(np.float32)
    nan = good.copy()
    nan[2] = np.nan
    same = np.array([33.0] * L + [44.0] * L, np.float32)                   # every used landmark equal: a = b = 0
    huge = (good * np.float32(1e30)).astype(np.float32)                   # a fixed-point coordinate leaves int32
    unused_nan = np.concatenate([good[:L], [np.nan], good[L:], [np.nan]]).astype(np.float32)   # an unused landmark is NaN
    assert ref.fit(nan, idx, u) is None and ref.fit(same, idx, u) is None
    assert ref.fit(good, idx, np.ones((L, 2))) is None                    # den == 0
    chips, c2f, f2c, valid = ref.face_chips([frame], [0] * 4, [good, nan, same, huge], idx, u, 40, 40)
    assert valid.tolist() == [True, False, False, False]
    assert not chips[1:].any() and not c2f[1:].any() and not f2c[1:].any()
    assert np.array_equal(chips[0], _cv2(frame, c2f[0], 40, 40))
    # an unused NaN landmark changes nothing
    x6 = unused_nan.reshape(2, L + 1)
    chips6, c2f6, _, valid6 = ref.face_chips([frame], [0], [x6.ravel()], idx, u, 40, 40)
    assert valid6[0] and np.array_equal(chips6[0], chips[0]) and np.array_equal(c2f6[0], c2f[0])


def test_int16_taps_only_matter_past_32767_px():
    """A tap coordinate outside int16 makes a face invalid only in a frame wider or taller than 32,767 px, where cv2 would
    saturate it; in smaller frames such taps are outside the frame and read 0 (cv2's remap takes frames below 32,767 px)."""
    M = _similarity(1.0, 0.0, 40000.0, 0.0)
    assert ref.taps(M, 8, 8, 32767, 10) is not None
    assert ref.taps(M, 8, 8, 32768, 10) is None
    assert ref.taps(_similarity(1.0, 0.0, 30000.0, 0.0), 8, 8, 40000, 10) is not None
    frame = np.full((4, 32766), 7, np.uint8)
    assert np.array_equal(ref.warp(frame, M, 8, 8), _cv2(frame, M, 8, 8))


def test_template():
    mean = np.array([-0.5, 0.0, 0.5, -0.5, 0.25, 0.5], np.float32)
    tm = ref.template(mean, 100, 50, padding=0.0)
    assert np.array_equal(tm, [[0.0, 0.0], [50.0, 37.5], [100.0, 50.0]])
    tm = ref.template(mean, 100, 50, padding=0.5, landmarks=[2, 0])
    assert np.array_equal(tm, [[75.0, 37.5], [25.0, 12.5]])

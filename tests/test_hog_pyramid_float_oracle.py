"""The resize rule of the float HOG pyramid (sd_hog_pyramid_float), on the CPU.

hog_resize_f32_ref.resize_f32 must equal cv2.resize(INTER_LINEAR) of float32 frames bit for bit, compared as int32 views, with
cv2's IPP switched off: IPP's own arithmetic differs from cv2's generic code by about 1.8e-5 relative.  That holds at every level
except exact 2x downscales on both axes, where cv2 switches to INTER_AREA and sums the four pixels in an order that depends on
the channel count and on SIMD column blocks; test_exact_2x_deviation pins how far the one linear rule is from it there."""
import numpy as np
import pytest

from hog_resize_f32_ref import level_size, resize_f32

cv2 = pytest.importorskip("cv2")

SCALES = [1.0, 0.5, 2.0, 1.5, 2 ** -0.2, 2 ** -0.6, 0.37, 0.2, 0.25, 3.0, 4.0, 2.37]
SIZES = [(97, 131), (120, 160), (45, 61), (64, 64), (33, 100)]


@pytest.fixture
def no_ipp():
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        yield
    finally:
        cv2.ipp.setUseIPP(was)


def _cv2(frame, lw, lh):
    return cv2.resize(frame, (lw, lh), interpolation=cv2.INTER_LINEAR).reshape((lh, lw) + frame.shape[2:])


def _bits_equal(a, b):
    """Equal as int32 views, except that NaNs made by arithmetic are equal to each other: their sign and payload come from
    the hardware and the compiler's operand order (x86 keeps the first operand's NaN, the H100 makes its canonical NaN), so
    they are no part of the rule.  Copied NaNs are compared by test_same_size_level_is_a_bit_copy."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    keep = ~np.isnan(a)
    return np.array_equal(a.view(np.int32)[keep], b.view(np.int32)[keep])


def _exact_2x(w, h, lw, lh):
    return w == 2 * lw and h == 2 * lh


def _frame(rng, h, w, c):
    return rng.uniform(-40.0, 300.0, (h, w, c)).astype(np.float32)


@pytest.mark.parametrize("c", [1, 2, 3, 4, 5, 16])
def test_rule_equals_cv2_off_exact_2x(no_ipp, c):
    rng = np.random.default_rng(100 + c)
    n = 0
    for h, w in SIZES:
        frame = _frame(rng, h, w, c)
        for s in SCALES:
            lw, lh = level_size(w, h, s)
            if _exact_2x(w, h, lw, lh):
                continue
            assert _bits_equal(resize_f32(frame, lw, lh), _cv2(frame, lw, lh)), (c, h, w, s)
            n += 1
    assert n >= 50


@pytest.mark.parametrize("c", [1, 3, 4])
def test_thin_and_single_pixel_frames(no_ipp, c):
    rng = np.random.default_rng(7 + c)
    for h, w in [(1, 1), (1, 9), (1, 40), (9, 1), (40, 1), (2, 1), (1, 2)]:
        frame = _frame(rng, h, w, c)
        for lw, lh in [(1, 1), (w, h), (3 * w, 2 * h), (max(1, w // 3), max(1, h // 3)), (4 * w, 4 * h), (w + 1, 1), (1, h + 1)]:
            assert _bits_equal(resize_f32(frame, lw, lh), _cv2(frame, lw, lh)), (c, h, w, lw, lh)


@pytest.mark.parametrize("c", [1, 3, 4, 5])
def test_exact_2x_on_one_axis_stays_linear(no_ipp, c):
    rng = np.random.default_rng(30 + c)
    for h, w in [(40, 64), (37, 90), (64, 31)]:
        frame = _frame(rng, h, w, c)
        for lw, lh in [(w // 2, h), (w, h // 2), (w // 2, h // 3), (w // 3, h // 2), (w // 2, (h + 1) // 2 + 1)]:
            assert not _exact_2x(w, h, lw, lh)
            assert _bits_equal(resize_f32(frame, lw, lh), _cv2(frame, lw, lh)), (c, h, w, lw, lh)


def _special_frame(rng, h, w, c):
    """Values cv2 must carry through taps of weight 0 and clamped border rows: NaN, +-inf, -0 and subnormals.  A level of the
    frame's width reads every right neighbour at weight 0, and a 3x downscale has fraction 0 in every column; upscales clamp the
    first and last rows with weights that do not sum to 1 in float."""
    f = _frame(rng, h, w, c)
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-41, -3e-39, np.float32(1.4e-45)], np.float32)
    m = rng.random((h, w, c)) < 0.08
    f[m] = rng.choice(specials, int(m.sum()))
    f[0, :, 0] = -0.0                                # a border row of -0
    f[-1, ::3, -1] = np.float32(2e-40)               # subnormals on the last row
    f[:, 1, :] = np.inf                              # column 1: the zero-weight right tap of column 0 at equal widths
    return f


def test_same_size_level_is_a_bit_copy(no_ipp):
    rng = np.random.default_rng(5)
    frame = _special_frame(rng, 21, 34, 3)
    frame[3, 4, 1] = np.array([0x7FC12345], np.uint32).view(np.float32)[0]     # a NaN payload
    frame[5, 6, 2] = np.array([0xFFA00001], np.uint32).view(np.float32)[0]     # a negative signalling NaN
    for got in (resize_f32(frame, 34, 21), _cv2(frame, 34, 21)):
        assert np.array_equal(got.view(np.int32), frame.view(np.int32))


@pytest.mark.parametrize("c", [1, 3, 4, 16])
def test_non_finite_and_subnormal_values(no_ipp, c):
    rng = np.random.default_rng(50 + c)
    skipped_differs = False
    for h, w in [(30, 45), (31, 60), (12, 12)]:
        frame = _special_frame(rng, h, w, c)
        for lw, lh in [(w, h), (w, h // 2 + 3), (w // 3, h // 3), (w // 3, h), (3 * w, 2 * h), (int(w * 0.6), int(h * 1.7)),
                       (w + 5, h - 1), (1, 1)]:
            want = _cv2(frame, lw, lh)
            assert _bits_equal(resize_f32(frame, lw, lh), want), (c, h, w, lw, lh)
            if not _bits_equal(resize_f32(frame, lw, lh, skip_zero_taps=True), want):
                skipped_differs = True
    # a kernel that leaves out zero-weight taps does not pass this test
    assert skipped_differs


def _rel(a, b):
    a, b = a.astype(np.float64), b.astype(np.float64)
    return np.abs(a - b) / np.maximum(np.abs(b), 1e-30)


@pytest.mark.parametrize("c", [1, 2, 3, 4, 5, 16])
def test_exact_2x_deviation(no_ipp, c):
    """At W = 2w and H = 2h cv2 uses INTER_AREA.  The linear rule gives ((a + b) + (c + d)) * 0.25 there: equal to cv2 at 4
    channels; at 1 channel equal except on the last w mod 4 columns; otherwise within one rounding."""
    rng = np.random.default_rng(70 + c)
    any_differs = False
    for h, w in [(120, 160), (64, 64), (46, 70), (18, 38), (720, 1280)] if c == 1 else [(120, 160), (46, 70), (18, 38)]:
        frame = rng.uniform(0.0, 255.0, (h, w, c)).astype(np.float32)
        lw, lh = w // 2, h // 2
        mine, want = resize_f32(frame, lw, lh), _cv2(frame, lw, lh)
        if c == 4:
            assert _bits_equal(mine, want), (h, w)
            continue
        if c == 1:
            head = 4 * (lw // 4)
            assert _bits_equal(mine[:, :head], want[:, :head]), (h, w)
        assert _rel(mine, want).max() <= 2.4e-7, (c, h, w)
        any_differs |= not _bits_equal(mine, want)
    if c != 4:
        assert any_differs                           # the deviation is real, not a stale note

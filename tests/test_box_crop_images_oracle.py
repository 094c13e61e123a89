"""The colour and float box crop of tests/box_crop_images_ref.py on the CPU: 8-bit crops at 1, 3 and 4 channels equal
cv2.copyMakeBorder(BORDER_CONSTANT, 0) + cv2.resize(INTER_LINEAR) channel by channel, and float crops equal cv2 of the padded
rectangle (IPP off, whose own arithmetic differs) except at exact 2x downscales (where cv2 switches to INTER_AREA), for boxes
inside the frame, past each edge, wholly outside it, and a rectangle of the crop's own size (a copy)."""
import numpy as np
import pytest

import box_crop_images_ref as ref
import synth
import track_ref


@pytest.fixture
def no_ipp():
    cv2 = pytest.importorskip("cv2")
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    try:
        yield cv2
    finally:
        cv2.ipp.setUseIPP(was)


def _frame(C, dtype, seed, H=83, W=121):
    g = np.stack([synth.smooth_images(1, H, W, seed=seed + c, sigma=1.0)[0] for c in range(C)], axis=-1)
    g = g[:, :, 0] if C == 1 else g
    return g.astype(np.float32) / np.float32(255) if dtype == np.float32 else g


def _boxes(H, W, fw, fh, cs):
    w, h = W // 3, H // 3
    return [(W // 3, H // 4, w, h),                 # inside
            (-w // 2, H // 3, w, h),                # past the left edge
            (W - w // 2, H // 3, w, h),             # past the right edge
            (W // 4, -h // 3, w, h),                # past the top
            (W // 4, H - h // 4, w, h),             # past the bottom
            (-3 * w, -3 * h, w, h),                 # wholly outside
            (5, 7, fw * cs, fh * cs)]               # context (fw + 2) cs x (fh + 2) cs: the crop's own size


def _cv2_crop(cv2, frame, box, fw, fh, cs):
    x, y, w, h = track_ref.context_rect(box, fw, fh)
    H, W = frame.shape[:2]
    pad = max(0, -x, -y, x + w - W, y + h - H)
    p = cv2.copyMakeBorder(frame, pad, pad, pad, pad, cv2.BORDER_CONSTANT, value=0)
    roi = np.ascontiguousarray(p[y + pad:y + pad + h, x + pad:x + pad + w])
    size = ((fw + 2) * cs, (fh + 2) * cs)
    if roi.ndim == 2:
        return cv2.resize(roi, size, interpolation=cv2.INTER_LINEAR)
    return np.stack([cv2.resize(np.ascontiguousarray(roi[:, :, c]), size, interpolation=cv2.INTER_LINEAR) for c in range(roi.shape[2])],
                    axis=-1)


@pytest.mark.parametrize("C", [1, 3, 4])
@pytest.mark.parametrize("fw,fh,cs", [(6, 6, 8), (5, 3, 4), (1, 1, 3)])
def test_u8_crop_equals_cv2_per_channel(oracle, C, fw, fh, cs):
    cv2 = pytest.importorskip("cv2")
    frame = _frame(C, np.uint8, fw + cs)
    for box in _boxes(*frame.shape[:2], fw, fh, cs):
        got = ref.box_crop(oracle, frame, box, fw, fh, cs)
        assert got.shape == ((fh + 2) * cs, (fw + 2) * cs) + ((C,) if C > 1 else ())
        assert np.array_equal(got, _cv2_crop(cv2, frame, box, fw, fh, cs)), box


@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("fw,fh,cs", [(6, 6, 8), (5, 3, 4), (1, 1, 3)])
def test_float_crop_equals_cv2_away_from_exact_2x(no_ipp, C, fw, fh, cs):
    cv2 = no_ipp
    frame = _frame(C, np.float32, fw + 2 * cs)
    for box in _boxes(*frame.shape[:2], fw, fh, cs):
        rect = track_ref.context_rect(box, fw, fh)
        got = ref.box_crop(None, frame, box, fw, fh, cs)
        assert got.dtype == np.float32
        if rect[2] == 2 * (fw + 2) * cs and rect[3] == 2 * (fh + 2) * cs:
            continue                                    # cv2's INTER_AREA switch, the documented exception
        assert np.array_equal(got.view(np.uint32), _cv2_crop(cv2, frame, box, fw, fh, cs).view(np.uint32)), box


def test_float_copy_case_is_a_bit_copy_with_zero_outside():
    fw, fh, cs = 2, 2, 2
    frame = np.full((10, 12), -0.0, np.float32)
    frame[3, 4] = np.float32(np.nan)
    box = (2, 2, 4, 4)                                  # e = (2, 2): the 8 x 8 rectangle at (0, 0) is the crop's size
    assert track_ref.context_rect(box, fw, fh) == (0, 0, 8, 8)
    got = ref.box_crop(None, frame, box, fw, fh, cs)
    assert np.array_equal(got.view(np.uint32), frame[:8, :8].view(np.uint32))
    out = ref.box_crop(None, frame, (-20, -20, 4, 4), fw, fh, cs)     # wholly outside: +0.0f everywhere
    assert out.shape == (8, 8) and not out.view(np.uint32).any()

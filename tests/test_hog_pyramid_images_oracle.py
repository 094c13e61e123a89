"""The resize rule of the colour HOG pyramid (sd_hog_pyramid_images), on the CPU.

Each channel of a level is oracle.resize_linear_u8 of that channel alone, the 8-bit INTER_LINEAR rule of the grey pyramid.  For
1, 3 and 4 channels that is cv2.resize of the whole frame at every level size used here, scales 0.5 and 2.0 included; for 2
channels cv2 takes another code path at exact 2x downscales and differs by 1 on some pixels, while the per-channel rule stays the
one the library uses.  The GPU tests pin the pyramid to this per-channel rule."""
import math

import numpy as np
import pytest

import synth

SCALES = [1.0, 0.5, 2.0, 1.5, 2 ** -0.2, 2 ** -0.6, 0.37, 0.2]
SIZES = [(97, 131), (120, 160), (45, 61), (64, 64)]


def _frame(h, w, c, seed):
    planes = [synth.smooth_images(1, h, w, seed=seed + 7 * k, sigma=1.0)[0] for k in range(c)]
    return np.ascontiguousarray(np.stack(planes, -1))


def per_channel(oracle, frame, lw, lh):
    """The library's rule: every channel resized on its own."""
    return np.stack([oracle.resize_linear_u8(frame[..., k], lw, lh) for k in range(frame.shape[2])], -1)


@pytest.mark.parametrize("c", [1, 3, 4])
def test_per_channel_rule_equals_cv2(oracle, c):
    cv2 = pytest.importorskip("cv2")
    for i, (h, w) in enumerate(SIZES):
        frame = _frame(h, w, c, seed=10 * c + i)
        for s in SCALES:
            lw, lh = math.floor(w * s + 0.5), math.floor(h * s + 0.5)
            want = cv2.resize(frame, (lw, lh), interpolation=cv2.INTER_LINEAR).reshape(lh, lw, c)
            assert np.array_equal(per_channel(oracle, frame, lw, lh), want), (c, h, w, s)


def test_two_channels_at_half_scale_differ_from_cv2(oracle):
    cv2 = pytest.importorskip("cv2")
    differs = 0
    for i, (h, w) in enumerate(SIZES):
        frame = _frame(h, w, 2, seed=90 + i)
        lw, lh = math.floor(w * 0.5 + 0.5), math.floor(h * 0.5 + 0.5)
        mine = per_channel(oracle, frame, lw, lh)
        # the rule does not depend on the channel count: channel k alone, or next to others, resizes the same
        for k in range(2):
            assert np.array_equal(mine[..., k], oracle.resize_linear_u8(frame[..., k], lw, lh))
        d = np.abs(cv2.resize(frame, (lw, lh), interpolation=cv2.INTER_LINEAR).astype(int) - mine.astype(int))
        assert d.max() <= 1
        differs += int(np.count_nonzero(d))
    assert differs > 0

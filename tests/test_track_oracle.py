"""The tracking rules on the CPU (tests/track_ref.py): the box crop equals cv2.resize of the zero-padded context rectangle for boxes
inside, across and outside the frame's edges; the face box of a set of landmarks on hand-computed cases, ties and degenerate
cases included; and box(align_mean(mean, B)) == B over many boxes with the rcr_22 mean."""
import os

import numpy as np
import pytest

import synth
import track_ref
from superviseddescent_b200 import api as sd

MODEL = os.path.join(os.path.dirname(__file__), "golden", "face_landmarks_model_rcr_22.bin")


def _boxes(rng, H, W, n):
    """Boxes inside the frame, across each edge and wholly outside it."""
    out = []
    for _ in range(n):
        w, h = int(rng.integers(4, W // 2)), int(rng.integers(4, H // 2))
        out.append((int(rng.integers(0, W - w)), int(rng.integers(0, H - h)), w, h))                # inside
        out.append((int(rng.integers(-w + 1, W - 1)), int(rng.integers(-h + 1, 0)), w, h))          # across the top
        out.append((int(rng.integers(W - w + 1, W)), int(rng.integers(0, H - h)), w, h))            # across the right edge
        out.append((int(rng.integers(-3 * w, -w - 1)), int(rng.integers(-h, H)), w, h))             # outside, left
        out.append((-w // 2, -h // 2, W + w, H + h))                                                 # larger than the frame
    return out


@pytest.mark.parametrize("fw,fh,cs", [(6, 6, 8), (5, 3, 4), (1, 1, 3), (4, 7, 6)])
def test_box_crop_equals_cv2_of_the_padded_roi(oracle, fw, fh, cs):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(fw * 100 + fh * 10 + cs)
    frame = synth.smooth_images(1, 97, 131, seed=fw + cs, sigma=1.0)[0]
    for box in _boxes(rng, 97, 131, 6):
        rect = track_ref.context_rect(box, fw, fh)
        roi = track_ref.padded_roi(frame, rect)
        assert roi.shape == (rect[3], rect[2])
        want = cv2.resize(roi, ((fw + 2) * cs, (fh + 2) * cs), interpolation=cv2.INTER_LINEAR)
        assert np.array_equal(track_ref.box_crop(oracle, frame, box, fw, fh, cs), want), box


def test_padded_roi_is_zero_outside_the_frame():
    frame = np.arange(12, dtype=np.uint8).reshape(3, 4) + 1
    roi = track_ref.padded_roi(frame, (-1, -2, 3, 4))
    assert roi.tolist() == [[0, 0, 0], [0, 0, 0], [0, 1, 2], [0, 5, 6]]
    assert not track_ref.padded_roi(frame, (10, 10, 2, 2)).any()
    # e = cvRound(w / fw), ties to even: 10 / 4 = 2.5 -> 2, 14 / 4 = 3.5 -> 4
    assert track_ref.context_rect((5, 6, 10, 14), 4, 4) == (3, 2, 14, 22)


def test_track_box_known_answers():
    mean = np.array([0.0, 1.0, 0.25, 0.0, 0.5, 1.0], np.float32)     # x in [0, 1], y in [0, 1]
    # landmarks of the box (10, 20, 100, 50): x = 100 m + 60, y = 50 m + 45
    assert track_ref.track_box([60, 160, 85, 45, 70, 95], mean) == (10, 20, 100, 50)
    # w = 2.5 -> 2 and bx = 0.5 - 0.5 * 2.5 = -0.75 -> -1; h = 3.5 -> 4 and by = 2 - 1.75 = 0.25 -> 0
    assert track_ref.track_box([0.5, 3.0, 1.0, 2.0, 3.0, 5.5], mean) == (-1, 0, 2, 4)
    # bx = 1.5 - 0.5 * 2 = 0.5 -> 0 and by = 2.5 - 0.5 * 2 = 1.5 -> 2 (ties to even)
    assert track_ref.track_box([1.5, 3.5, 2.0, 2.5, 3.0, 4.5], mean) == (0, 2, 2, 2)
    # degenerate: collapsed (w = 0), w rounding below 1, a NaN, an extent past int32, a mean without extent
    assert track_ref.track_box([5, 5, 5, 1, 2, 3], mean) is None
    assert track_ref.track_box([0, 0.49, 0.2, 0, 1, 2], mean) is None
    assert track_ref.track_box([0, 1, np.nan, 0, 1, 2], mean) is None
    assert track_ref.track_box([0, 3e9, 1, 0, 1, 2], mean) is None
    assert track_ref.track_box([0, 1, 2, 0, 1, 2], np.zeros(6, np.float32)) is None
    # w = 0.5 rounds to 0 (ties to even): degenerate; w = 1.5 rounds to 2
    assert track_ref.track_box([0, 0.5, 0.25, 0, 2, 1], mean) is None
    assert track_ref.track_box([0, 1.5, 0.25, 0, 2, 1], mean) == (-1, -1, 2, 2)


def test_box_of_align_mean_is_the_box(oracle):
    mean = oracle.Model(MODEL).mean
    rng = np.random.default_rng(5)
    boxes = [(int(rng.integers(-500, 2000)), int(rng.integers(-500, 2000)), int(rng.integers(20, 800)), int(rng.integers(20, 800)))
             for _ in range(3000)]
    boxes += [(x, y, s, s) for x in (-7, 0, 13, 1279) for y in (-3, 0, 719) for s in (12, 24, 64, 100, 333, 720)]
    for b in boxes:
        x0 = sd.align_mean(mean, b)
        assert np.array_equal(x0, oracle.align_mean(mean, b))
        assert track_ref.track_box(x0, mean) == b, b

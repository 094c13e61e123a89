"""The detection rule's numpy restatement (hog_detect_ref.py), checked three ways on the CPU:

- its greedy suppression against torchvision.ops.nms on random integer boxes whose IoU is not within 1e-6 of the threshold (the
  two rules then agree exactly); skipped when torchvision does not import;
- a case worked by hand: positions left of and above the frame (x - pad_x < 0, floor division of negative numerators), level
  ratios with W / level_w != 1 / s, ties in the order, and suppression;
- the box rule against hog_pyramid_shape's levels and the header's mapping of a score to pixels, (x - pad_x) * cell_size * W /
  level_w, rounded half up in exact rational arithmetic."""
from fractions import Fraction

import numpy as np
import pytest

import hog_detect_ref as R


def _iou64(b, j, k):
    iw = max(0, min(b[2][j], b[2][k]) - max(b[0][j], b[0][k]))
    ih = max(0, min(b[3][j], b[3][k]) - max(b[1][j], b[1][k]))
    inter = iw * ih
    union = (b[2][j] - b[0][j]) * (b[3][j] - b[1][j]) + (b[2][k] - b[0][k]) * (b[3][k] - b[1][k]) - inter
    return inter / union if union else 0.0


@pytest.mark.parametrize("seed", range(6))
def test_suppression_matches_torchvision_nms(seed):
    tv = pytest.importorskip("torchvision")
    import torch
    rng = np.random.default_rng(seed)
    n = 300
    thr = [0.0, 0.3, 0.5, 0.7][seed % 4]
    x0, y0 = rng.integers(-20, 80, n), rng.integers(-20, 80, n)
    x1, y1 = x0 + rng.integers(0, 40, n), y0 + rng.integers(0, 40, n)        # some boxes of zero width or height
    b = [x0.astype(np.int64), y0.astype(np.int64), x1.astype(np.int64), y1.astype(np.int64)]
    # drop boxes whose IoU with any other lies within 1e-6 of the threshold: the float division of torchvision and the
    # multiplication of the rule may then disagree (an IoU of exactly 0 is never above a threshold in either)
    keep = []
    for j in range(n):
        if all(abs(_iou64(b, j, k) - thr) > 1e-6 or _iou64(b, j, k) == 0 for k in keep):
            keep.append(j)
    b = [v[keep] for v in b]
    m = len(keep)
    scores = np.linspace(1.0, 0.0, m)                                          # distinct, in order
    got = R.suppress(*b, thr, m)
    ref = tv.ops.nms(torch.from_numpy(np.stack(b, 1).astype(np.float64)), torch.from_numpy(scores), thr).numpy()
    print(f"seed {seed}: {m} boxes, threshold {thr}, kept {got.size}")
    assert np.array_equal(got, ref)
    # overlap = 1 keeps everything, and the cap stops early
    assert R.suppress(*b, 1.0, m).size == m
    assert np.array_equal(R.suppress(*b, thr, 5), got[:5])


def test_round_half_up_floors():
    assert [R.rh(n, 10) for n in (-26, -25, -15, -14, 0, 5, 14, 15, 25)] == [-3, -2, -1, -1, 0, 1, 1, 2, 3]
    assert R.rh(np.int64(-15), np.int64(10)) == -1


def test_hand_worked_boxes():
    # a 101 x 49 frame at scale 0.3: level 30 x 15 px (floor(30.3 + 0.5), floor(14.7 + 0.5)), so W / level_w = 3.3667 and
    # H / level_h = 3.2667, not 1 / 0.3.  cell 8, filter 3 x 2 cells, pads (2, 1): sx = 808, sy = 392.
    m = R.ScoreMap(0, 4, 101, 49, 30, 15, np.zeros((1, 4, 6), np.float32))
    # (0, 0): x0 = rh(-1616, 30) = -54 (-53.87), x1 = rh(808, 30) = 27 (26.93), y0 = rh(-392, 15) = -26 (-26.13),
    #         y1 = rh(392, 15) = 26 (26.13)
    # (5, 3): x0 = rh(2424, 30) = 81 (80.8), x1 = rh(4848, 30) = 162 (161.6), y0 = rh(784, 15) = 52 (52.27),
    #         y1 = rh(1568, 15) = 105 (104.53)
    got = R.boxes([0, 5], [0, 3], m, 8, 3, 2, 2, 1)
    assert [list(map(int, v)) for v in got] == [[-54, 81], [-26, 52], [27, 162], [26, 105]]

    s = np.zeros((2, 4, 6), np.float32)
    s[0, 0, 0] = 3.0
    s[1, 3, 5] = 3.0               # ties with (0, 0, 0): enumeration order puts q = 0 first
    s[0, 1, 1] = -0.0
    s[1, 1, 1] = 0.0               # -0 == +0: enumeration order again
    s[0, 2, 2] = np.nan            # never a candidate
    out, above = R.detections([R.ScoreMap(0, 4, 101, 49, 30, 15, s)], 2, 8, 3, 2, 2, 1, -1.0, 1.0, 64, 64)
    assert list(above) == [48 - 1, 0] and out[1].shape == (0, R.FIELDS)
    first = out[0][:4]
    assert [tuple(r[[5, 7, 8]]) for r in first] == [(0, 0, 0), (1, 5, 3), (0, 1, 0), (0, 2, 0)]
    assert tuple(first[0, :4]) == (-54, -26, 81, 52) and tuple(first[1, :4]) == (81, 52, 81, 53)
    assert first[0, 4] == np.float32(3.0).view(np.int32) and first[0, 6] == 4


def test_hand_worked_order_and_suppression():
    # an unscaled 40 x 40 frame, cell 4, 2 x 2-cell filter: position (x, y) is the box (4x, 4y, 8, 8)
    s = np.zeros((1, 3, 3), np.float32)
    s[0, 0, 0], s[0, 1, 1], s[0, 2, 2] = 1.0, 2.0, 2.0
    maps = [R.ScoreMap(0, 0, 40, 40, 40, 40, s)]
    out, _ = R.detections(maps, 1, 4, 2, 2, 0, 0, 0.5, 0.5, 16, 16)
    assert [tuple(r) for r in out[0][:, [0, 1, 2, 3, 7, 8]]] == [(4, 4, 8, 8, 1, 1), (8, 8, 8, 8, 2, 2), (0, 0, 8, 8, 0, 0)]
    # IoU of (1, 1) with either neighbour is 16 / 112 = 0.143: suppressed at 0.1, kept at 0.5 (above)
    out, _ = R.detections(maps, 1, 4, 2, 2, 0, 0, 0.5, 0.1, 16, 16)
    assert [tuple(r) for r in out[0][:, [7, 8]]] == [(1, 1)]
    # the cap: only the first two candidates reach suppression
    out, above = R.detections(maps, 1, 4, 2, 2, 0, 0, 0.5, 0.5, 2, 2)
    assert above[0] == 3 and [tuple(r) for r in out[0][:, [7, 8]]] == [(1, 1), (2, 2)]


@pytest.mark.parametrize("seed", range(4))
def test_boxes_agree_with_pyramid_levels(seed):
    from superviseddescent_b200 import api
    rng = np.random.default_rng(seed)
    for _ in range(20):
        W, H = int(rng.integers(20, 1500)), int(rng.integers(20, 1000))
        s = float(rng.choice([1.0, 0.5, 2 ** -0.25, 0.37, 1.7, 2 ** (-rng.integers(1, 12) / 5)]))
        cell = int(rng.choice([4, 6, 8]))
        (lw, lh), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, cell, 9, 1)
        if hh == 0:
            continue
        fw, fh = int(rng.integers(1, min(hw, 8) + 1)), int(rng.integers(1, min(hh, 8) + 1))
        px, py = int(rng.integers(0, fw)), int(rng.integers(0, fh))
        m = R.ScoreMap(0, 0, W, H, lw, lh, None)
        xs = np.arange(hw + 2 * px - fw + 1)
        ys = np.arange(hh + 2 * py - fh + 1)
        x0, _, x1, _ = R.boxes(xs, np.zeros_like(xs), m, cell, fw, fh, px, py)
        _, y0, _, y1 = R.boxes(np.zeros_like(ys), ys, m, cell, fw, fh, px, py)
        half = Fraction(1, 2)
        for x, a, b in zip(xs, x0, x1):
            assert a == int(np.floor(Fraction(int(x - px) * cell * W, lw) + half))
            assert b == int(np.floor(Fraction(int(x - px + fw) * cell * W, lw) + half))
        for y, a, b in zip(ys, y0, y1):
            assert a == int(np.floor(Fraction(int(y - py) * cell * H, lh) + half))
            assert b == int(np.floor(Fraction(int(y - py + fh) * cell * H, lh) + half))
        # a filter over every cell of the level, unpadded, spans the frame to within half a cell of the level
        full = R.boxes([0], [0], m, cell, hw, hh, 0, 0)
        assert full[0][0] == 0 and full[1][0] == 0
        assert abs(int(full[2][0]) - W) <= Fraction(cell * W, 2 * lw) + 1 and abs(int(full[3][0]) - H) <= Fraction(cell * H, 2 * lh) + 1

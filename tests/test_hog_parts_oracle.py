"""CPU checks of hog_parts_ref, the restatement the GPU part-model tests compare against bit for bit.

The restated transform agrees with an independent float64 brute force over every (dx, dy): values within the rounding of two
float32 subtractions, placements equal wherever the float64 maximum is unique by more than that rounding.  Hand-worked 1-D and
2-D cases pin the separable tie rule, NaN and infinities; R = 0 is the identity; the assembly adds parts in order and gives -inf
for an anchor outside the part map; a part's box follows sd_hog_detections' rule at the part level."""
import numpy as np
import pytest

import hog_parts_ref as ref

EPS = np.float64(2.0 ** -24)


def _random_case(rng, h, w, R, integer):
    if integer:
        s = rng.integers(-4, 5, (h, w)).astype(np.float32)
        d = rng.integers(0, 3, 4).astype(np.float32)
        d[[1, 3]] = rng.integers(-2, 3, 2)
    else:
        s = rng.normal(0, 3, (h, w)).astype(np.float32)
        d = np.array([rng.uniform(0, 0.5), rng.normal(0, 0.3), rng.uniform(0, 0.5), rng.normal(0, 0.3)], np.float32)
    return s, d


@pytest.mark.parametrize("h,w,R", [(1, 1, 0), (1, 7, 2), (6, 1, 3), (9, 11, 1), (12, 10, 4), (5, 6, 8), (17, 13, 5)])
@pytest.mark.parametrize("integer", [False, True])
def test_restatement_matches_float64_brute_force(h, w, R, integer):
    rng = np.random.default_rng(h * 100 + w * 10 + R + integer)
    for _ in range(3):
        s, d = _random_case(rng, h, w, R, integer)
        D, place = ref.transform(s, d, R)
        best, gap, where = ref.brute64(s, d, R)
        cx, cy = ref.cost_tables(d, R)
        bar = 2 * EPS * (np.abs(s).max() + np.abs(cx).max() + np.abs(cy).max())
        assert np.all(np.abs(D.astype(np.float64) - best) <= bar)
        unique = gap > 2 * bar
        assert np.array_equal(place[unique], where[unique].astype(np.int32))
        if integer:                       # exact arithmetic: the value is the float64 maximum itself
            assert np.array_equal(D.astype(np.float64), best)
        # the placement reaches the value: the candidate at the placement gives D in the rule's arithmetic
        v, u = np.nonzero(place[..., 0] >= 0)
        pu, pv = place[v, u, 0], place[v, u, 1]
        cand = (s[pv, pu] - cx[pu - u + R]) - cy[pv - v + R]
        assert np.array_equal(cand, D[v, u])


def test_one_row_by_hand():
    D, place = ref.transform(np.array([[1, 3, 1]], np.float32), [1, 0, 1, 0], 1)
    assert D.tolist() == [[2, 3, 2]]
    assert place[0, :, 0].tolist() == [1, 1, 1] and place[0, :, 1].tolist() == [0, 0, 0]
    # equal candidates: the smallest displacement wins
    D, place = ref.transform(np.array([[2, 2, 2]], np.float32), [0, 0, 0, 0], 1)
    assert D.tolist() == [[2, 2, 2]] and place[0, :, 0].tolist() == [0, 0, 1]
    # a linear term moves the choice: w1 = -1 makes +dx cheaper, each step gains 1, but the quadratic term costs 1 per unit
    D, place = ref.transform(np.array([[0, 0, 0, 0]], np.float32), [1, -1, 0, 0], 2)
    # at u = 0: d = 0 -> 0, d = 1 -> 0, d = 2 -> -2: tie between 0 and 1 -> 0
    assert place[0, :, 0].tolist() == [0, 1, 2, 3] and D.tolist() == [[0, 0, 0, 0]]


def test_two_dimensions_by_hand_with_ties():
    s = np.zeros((3, 3), np.float32)
    D, place = ref.transform(s, [0, 0, 0, 0], 1)
    assert np.all(D == 0)
    # the smallest e first, then the smallest d in that row
    assert place[1, 1].tolist() == [0, 0] and place[0, 0].tolist() == [0, 0] and place[2, 2].tolist() == [1, 1]
    s[2, 0] = 1
    D, place = ref.transform(s, [0.25, 0, 0.5, 0], 1)
    assert D[1, 1] == np.float32(0.25) and place[1, 1].tolist() == [0, 2]
    assert D[2, 1] == np.float32(0.75) and place[2, 1].tolist() == [0, 2]


def test_nan_and_infinities():
    s = np.array([[np.nan, np.nan, np.nan], [np.nan, np.inf, -np.inf]], np.float32)
    D, place = ref.transform(s, [1, 0, 1, 0], 1)
    assert np.all(np.isposinf(D[:, :3]))                      # +inf is within reach of every position
    s = np.full((2, 4), np.nan, np.float32)
    s[1, 3] = -np.inf
    D, place = ref.transform(s, [1, 0, 1, 0], 1)
    assert np.all(np.isneginf(D))
    # row 0 at u = 0..1 has no non-NaN candidate in X, and neither does row 1: no placement
    assert place[0, 0].tolist() == [-1, -1] and place[1, 0].tolist() == [-1, -1]
    # pass Y takes row 0's -inf first (the smallest e), and row 0 chose nothing in X: no placement
    assert place[1, 3].tolist() == [-1, -1]
    # a -inf candidate is a candidate: the first non-NaN one is taken
    D, place = ref.transform(np.array([[np.nan, -np.inf, -np.inf]], np.float32), [1, 0, 1, 0], 1)
    assert np.all(np.isneginf(D)) and place[0, :, 0].tolist() == [1, 1, 1] and place[0, :, 1].tolist() == [0, 0, 0]


@pytest.mark.parametrize("h,w", [(1, 1), (4, 7), (9, 3)])
def test_zero_displacement_is_the_identity(h, w):
    s = np.random.default_rng(h * w).normal(0, 1, (h, w)).astype(np.float32)
    D, place = ref.transform(s, [3.5, -1.25, 0.5, 2.0], 0)
    assert np.array_equal(D.view(np.int32), s.view(np.int32))
    v, u = np.mgrid[0:h, 0:w]
    assert np.array_equal(place[..., 0], u) and np.array_equal(place[..., 1], v)


def test_assembly_order_and_outside_anchors():
    root = np.array([[[1e8, 0.5]]], np.float32)               # Q = 1, oh = 1, ow = 2
    D = np.zeros((2, 3, 5), np.float32)
    D[0] = 1.0
    D[1] = -1e8
    anchors = np.array([[[0, 0], [2, 1]]])
    out = ref.part_scores(root, D, anchors, (0, 0), (0, 0))
    # x = 0: ((1e8 + 1) + -1e8) = 0 in float32 (1e8 + 1 rounds to 1e8); x = 1: part 1 at u0 = 4, v0 = 1
    assert out[0, 0, 0] == np.float32(np.float32(np.float32(1e8) + np.float32(1)) + np.float32(-1e8))
    assert out[0, 0, 0] == 0
    assert out[0, 0, 1] == np.float32(np.float32(0.5 + 1.0) - np.float32(1e8))
    anchors = np.array([[[0, 0], [3, 1]]])                      # x = 1: part 1 at u0 = 5 is outside
    out = ref.part_scores(root, D, anchors, (0, 0), (0, 0))
    assert np.isneginf(out[0, 0, 1]) and out[0, 0, 0] == 0
    assert np.all(np.isneginf(ref.part_scores(root, None, anchors, (0, 0), (0, 0))))


def test_part_boxes_follow_the_detection_rule():
    D = np.zeros((1, 4, 6), np.float32)
    place = np.zeros((1, 4, 6, 2), np.int32)
    place[0, 2, 3] = (4, 1)
    pmap = {"D": D, "place": place, "frame_w": 100, "frame_h": 60, "part_level_w": 50, "part_level_h": 30}
    rec = np.array([0, 0, 0, 0, 0, 0, 0, 1, 1], np.int32)      # q 0 at score position (1, 1)
    rows = ref.placements(rec, pmap, np.array([[[1, 0]]]), (0, 0), (0, 0), (2, 2), 4)
    # anchor (2 * 1 + 1, 2 * 1 + 0) = (3, 2) -> placement (4, 1); x0 = rh(4 * 4 * 100, 50) = 32, x1 = rh(6 * 400, 50) = 48
    assert rows[0].tolist() == [4, 1, 0, 32, 8, 16, 16]
    rows = ref.placements(rec, pmap, np.array([[[9, 0]]]), (0, 0), (0, 0), (2, 2), 4)
    assert rows[0, :2].tolist() == [-1, -1] and rows[0, 3:].tolist() == [0, 0, 0, 0]
    assert np.isneginf(rows[0, 2:3].view(np.float32)[0])

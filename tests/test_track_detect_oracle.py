"""The association and merge restatement of tests/track_detect_ref.py against brute force: an overlap matrix in int64 numpy over
every pair of boxes, the association as a mask over every (detection, row) pair, and the merge as the one subset of alive rows
in which a row is kept iff no kept row before it in the order (old first, score key descending, row index) overlaps it, found
by trying every subset.  Cases: seeded boxes of a few frames among many, IoU exactly at the threshold as a rational (strict: not
dropped), equal scores (row order decides), -0 against +0, and track_overlap 0 and 1."""
import itertools

import numpy as np
import pytest

import track_detect_ref as ref


def _overlap_matrix(a, b, t):
    a, b = np.asarray(a, np.int64).reshape(-1, 4), np.asarray(b, np.int64).reshape(-1, 4)
    iw = np.minimum(a[:, None, 0] + a[:, None, 2], b[None, :, 0] + b[None, :, 2]) - np.maximum(a[:, None, 0], b[None, :, 0])
    ih = np.minimum(a[:, None, 1] + a[:, None, 3], b[None, :, 1] + b[None, :, 3]) - np.maximum(a[:, None, 1], b[None, :, 1])
    inter = np.where((iw > 0) & (ih > 0), iw * ih, 0)
    union = (a[:, 2] * a[:, 3])[:, None] + (b[:, 2] * b[:, 3])[None, :] - inter
    return inter.astype(np.float64) > np.float64(t) * union.astype(np.float64)


def _score_key(s):
    b = np.where(np.asarray(s, np.float32) == 0, np.float32(0), np.asarray(s, np.float32)).view(np.uint32).astype(np.uint64)
    return np.where(b & 0x80000000, ~b & 0xFFFFFFFF, b | 0x80000000)


def _brute_merge(frame, boxes, scores, alive, T, t):
    out = np.array(alive, bool).copy()
    ov = _overlap_matrix(boxes, boxes, t)
    rows_all = np.arange(len(frame))
    prio = (((rows_all < T).astype(np.uint64) << np.uint64(63)) | (_score_key(scores) << np.uint64(31))
            | (np.uint64(0x7FFFFFFF) - rows_all.astype(np.uint64)))
    for f in np.unique(np.asarray(frame)[out]):
        rows = [r for r in rows_all if out[r] and frame[r] == f]
        found = []
        for bits in itertools.product([False, True], repeat=len(rows)):
            kept = {r for r, b in zip(rows, bits) if b}
            if all((r in kept) == (not any(prio[k] > prio[r] and ov[k, r] for k in kept)) for r in rows):
                found.append(kept)
        assert len(found) == 1
        for r in rows:
            out[r] = r in found[0]
    return out


def _brute_associate(det_frame, det_boxes, row_frame, row_boxes, alive, t):
    ov = _overlap_matrix(det_boxes, row_boxes, t)
    same = np.asarray(det_frame)[:, None] == np.asarray(row_frame)[None, :]
    return ~(ov & same & np.asarray(alive, bool)[None, :]).any(1)


def _seeded(seed, n_rows, n_frames, frames_used):
    rng = np.random.default_rng(seed)
    frame = rng.choice(frames_used, n_rows).astype(np.int32)
    xy = rng.integers(0, 60, (n_rows, 2))
    wh = rng.integers(8, 40, (n_rows, 2))
    boxes = np.concatenate([xy, wh], 1).astype(np.int32)
    scores = rng.choice(np.array([-0.0, 0.0, 0.5, 0.5, 1.25, -2.0, 3.0], np.float32), n_rows)
    alive = rng.random(n_rows) < 0.8
    return frame, boxes, scores, alive


@pytest.mark.parametrize("t", [0.0, 0.3, 0.5, 1.0])
@pytest.mark.parametrize("seed", range(6))
def test_merge_and_association_match_brute_force(seed, t):
    frame, boxes, scores, alive = _seeded(seed, 24, 1000, [3, 500, 999])
    T = 14
    got = ref.merge(frame, boxes, scores, alive, T, t)
    assert np.array_equal(got, _brute_merge(frame, boxes, scores, alive, T, t))
    assert not (got & ~alive).any()
    if t == 1.0:
        assert np.array_equal(got, alive)
    dframe, dboxes, _, _ = _seeded(seed + 100, 30, 1000, [3, 500, 7])
    keep = ref.associate(dframe, dboxes, frame[:T], boxes[:T], alive[:T], t)
    assert np.array_equal(keep, _brute_associate(dframe, dboxes, frame[:T], boxes[:T], alive[:T], t))
    if t == 1.0:
        assert keep.all()
    assert keep[dframe == 7].all()                                       # no row lies in frame 7


def test_overlap_at_the_threshold_is_not_an_overlap():
    # inter 50, union 100: IoU 1/2 exactly
    a, b = (0, 0, 10, 10), (0, 5, 10, 5)
    assert not ref.overlap(a, b, 0.5) and ref.overlap(a, b, np.nextafter(0.5, 0))
    # inter 20, union 60: the rule compares in float64, where (1 / 3) * 60 rounds to 20.0
    a, b = (0, 0, 10, 4), (5, 0, 10, 4)
    assert not ref.overlap(a, b, 1 / 3) and ref.overlap(a, b, 0.33)
    assert ref.overlap(a, b, 0.0) and not ref.overlap((0, 0, 5, 5), (5, 0, 5, 5), 0.0)   # touching edges do not meet
    keep = ref.associate([0], [(0, 5, 10, 5)], [0], [(0, 0, 10, 10)], [True], 0.5)
    assert keep.tolist() == [True]


def test_merge_order_rules():
    boxes = np.array([(0, 0, 10, 10)] * 4, np.int32)
    frame = np.zeros(4, np.int32)
    # equal scores: the lower row wins; -0 and +0 are equal scores
    assert ref.merge(frame, boxes, np.float32([1, 1, 1, 1]), [True] * 4, 4, 0.5).tolist() == [True, False, False, False]
    assert ref.merge(frame, boxes, np.float32([-0.0, 0.0, -1, -1]), [True] * 4, 4, 0.5).tolist() == [True, False, False, False]
    assert ref.merge(frame, boxes, np.float32([0.0, -0.0, -1, -1]), [False, True, True, True], 4, 0.5).tolist() == [False, True, False, False]
    # the higher score wins among old rows, and an old row beats any new one
    assert ref.merge(frame, boxes, np.float32([1, 2, 5, 9]), [True] * 4, 2, 0.5).tolist() == [False, True, False, False]
    # rows of other frames never meet
    assert ref.merge(np.arange(4), boxes, np.float32([1, 2, 5, 9]), [True] * 4, 2, 0.0).all()

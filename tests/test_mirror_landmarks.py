"""The landmark correspondence of mirrored samples (mirror_permutation, mirror_landmarks, mirror_box): ibug-68's left-right pairs,
a known answer on the rcr_22 model's landmark list, the refusal of a list without a partner, and known answers for the landmark and
box mirrors.  CPU only."""
import numpy as np
import pytest

from superviseddescent_b200 import api as sd

IBUG68 = [str(i) for i in range(1, 69)]
FIXED = {9, 28, 29, 30, 31, 34, 52, 58, 63, 67}


def test_ibug68_permutation_is_an_involution_with_the_listed_fixed_points():
    perm = sd.mirror_permutation(IBUG68)
    assert sorted(perm.tolist()) == list(range(68))
    assert np.array_equal(perm[perm], np.arange(68))
    assert {i + 1 for i in range(68) if perm[i] == i} == FIXED
    pairs = {(1, 17), (8, 10), (18, 27), (22, 23), (32, 36), (33, 35), (37, 46), (38, 45), (39, 44), (40, 43), (41, 48), (42, 47),
             (49, 55), (50, 54), (51, 53), (56, 60), (57, 59), (61, 65), (62, 64), (66, 68)}
    for a, b in pairs:
        assert perm[a - 1] == b - 1 and perm[b - 1] == a - 1, (a, b)
    # the jaw line runs 1..17 and its mirror 17..1
    assert perm[:17].tolist() == list(range(16, -1, -1))


def test_rcr22_model_list_known_answer(oracle, golden):
    ids = oracle.Model(golden.model_path).landmark_ids
    assert ids == ['9', '31', '32', '36', '37', '38', '39', '40', '41', '42', '43', '44', '45', '46', '47', '48', '49', '52', '55',
                   '58', '63', '67']
    perm = sd.mirror_permutation(ids)
    assert perm.tolist() == [0, 1, 3, 2, 13, 12, 11, 10, 15, 14, 7, 6, 5, 4, 9, 8, 18, 17, 16, 19, 20, 21]


@pytest.mark.parametrize("ids", [["37", "38", "9"], ["49", "52"], ["1", "x"], ["0"], ["69"]])
def test_missing_partner_or_foreign_id_raises(ids):
    with pytest.raises(ValueError):
        sd.mirror_permutation(ids)


def test_mirror_box_known_answer():
    assert sd.mirror_box((10, 20, 30, 40), 100) == (60, 20, 30, 40)
    assert sd.mirror_box((0, 0, 7, 5), 7) == (0, 0, 7, 5)
    assert sd.mirror_box((-5, 3, 10, 10), 21) == (16, 3, 10, 10)


def test_mirror_landmarks_known_answer():
    perm = sd.mirror_permutation(["37", "46", "31"])
    assert perm.tolist() == [1, 0, 2]
    x = np.array([[10.0, 50.0, 30.5, 1.0, 2.0, 3.0],
                  [0.0, 99.0, 49.5, 7.0, 8.0, 9.0]], dtype=np.float32)
    got = sd.mirror_landmarks(x, [100, 64], perm)
    want = np.array([[49.0, 89.0, 68.5, 2.0, 1.0, 3.0],
                     [-36.0, 63.0, 13.5, 8.0, 7.0, 9.0]], dtype=np.float32)
    assert got.dtype == np.float32 and np.array_equal(got, want)
    # one width for all rows, one row, and mirroring twice gives the landmarks back
    assert np.array_equal(sd.mirror_landmarks(x[0], 100, perm), want[0])
    assert np.array_equal(sd.mirror_landmarks(sd.mirror_landmarks(x, 100, perm), 100, perm), x)
    with pytest.raises(ValueError):
        sd.mirror_landmarks(x, 100, [0, 1])

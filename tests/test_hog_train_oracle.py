"""The host-only parts of the HOG filter trainer and its float64 oracles, without a GPU.

- sd_hog_box_windows (api.hog_box_windows) equals the numpy restatement (hog_train_ref.box_windows) on every box of a sweep over
  frame sizes, scales, pads, cell sizes and filter sides, with boxes partly outside the frame and boxes no window reaches.
- Exact IoU ties go to the lower level, then y, then x.
- The restatement's boxes are hog_detect_ref's box rule.
- The float64 squared-hinge Newton reference reaches the optimum: scipy's minimize on the same objective agrees, and the KKT
  condition (a zero gradient of the differentiable f) holds.
- Every refusal of the host-only call."""
import numpy as np
import pytest
import scipy.optimize as so

import hog_detect_ref as DR
import hog_train_ref as T
from superviseddescent_b200 import api
from superviseddescent_b200._capi import SdError


def _levels(W, H, scales, cell, K=9, variant=1):
    return [api.hog_pyramid_shape(W, H, s, cell, K, variant) for s in scales]


SWEEP = [  # (W, H, scales, cell, fw, fh, pad_x, pad_y, overlap)
    (160, 120, [1.0, 0.8, 0.63], 8, 6, 6, 0, 0, 0.5),
    (200, 90, [1.3, 1.0, 0.7], 4, 5, 3, 2, 1, 0.5),
    (97, 131, [2.0, 1.0, 0.5], 6, 4, 4, 3, 0, 0.3),
    (64, 64, [1.0], 8, 8, 8, 0, 0, 0.0),
    (321, 77, [0.9, 0.45, 0.3], 5, 7, 2, 0, 1, 0.7),
]


def _boxes(rng, W, H, n=24):
    b = []
    for _ in range(n):
        w, h = int(rng.integers(4, max(5, W))), int(rng.integers(4, max(5, H)))
        x, y = int(rng.integers(-w // 2, W)), int(rng.integers(-h // 2, H))
        b.append((x, y, w, h))
    b += [(W + 50, H + 50, 10, 10), (-400, -400, 20, 20), (0, 0, 1, 1), (-5, -5, W + 10, H + 10)]   # none reach, tiny, covering
    return np.asarray(b, np.int32)


@pytest.mark.parametrize("case", range(len(SWEEP)))
def test_box_windows_equal_the_restatement(case):
    W, H, scales, cell, fw, fh, px, py, ov = SWEEP[case]
    rng = np.random.default_rng(case)
    boxes = _boxes(rng, W, H)
    got, iou = api.hog_box_windows(W, H, boxes, scales, (fw, fh), cell, 9, 1, pad=(px, py), positive_overlap=ov)
    ref, iou_ref = T.box_windows(W, H, boxes, _levels(W, H, scales, cell), cell, fw, fh, px, py, ov)
    print(f"case {case}: {int((got[:, 0] >= 0).sum())} of {len(boxes)} boxes assigned, best IoU {iou.max():.3f}")
    assert np.array_equal(got, ref)
    assert np.array_equal(iou, iou_ref)


def test_exact_ties_follow_level_then_y_then_x():
    # a box between two windows of one level: equal IoU to the left and right window -> the lower x; above and below -> lower y
    W = H = 128
    cell, fw, fh = 8, 4, 4
    scales = [1.0, 1.0]                                   # two identical levels: every tie across them goes to level 0
    box = np.asarray([[4, 0, 32, 32], [0, 4, 32, 32], [4, 4, 32, 32], [8, 8, 32, 32]], np.int32)
    got, iou = api.hog_box_windows(W, H, box, scales, (fw, fh), cell, 9, 1, positive_overlap=0.0)
    ref, _ = T.box_windows(W, H, box, _levels(W, H, scales, cell), cell, fw, fh, 0, 0, 0.0)
    assert np.array_equal(got, ref)
    assert got[0].tolist() == [0, 0, 0]                   # x = 0 and x = 1 tie (IoU 28 / 36 each)
    assert got[1].tolist() == [0, 0, 0]                   # y = 0 and y = 1 tie
    assert got[2].tolist() == [0, 0, 0]
    assert got[3].tolist() == [0, 1, 1] and iou[3] == 1.0


def test_restated_boxes_are_the_detection_box_rule():
    W, H, s, cell, fw, fh, px, py = 211, 143, 0.77, 6, 5, 4, 2, 3
    (lw, lh), (_, hh, hw) = api.hog_pyramid_shape(W, H, s, cell, 9, 1)
    oh, ow = hh + 2 * py - fh + 1, hw + 2 * px - fw + 1
    m = DR.ScoreMap(0, 0, W, H, lw, lh, np.zeros((1, oh, ow), np.float32))
    x, y = np.meshgrid(np.arange(ow), np.arange(oh))
    b = DR.boxes(x.ravel(), y.ravel(), m, cell, fw, fh, px, py)
    # a box equal to a window's box is assigned exactly that window at IoU 1
    k = int(np.flatnonzero((x.ravel() == 3) & (y.ravel() == 2))[0])
    box = np.asarray([[b[0][k], b[1][k], b[2][k] - b[0][k], b[3][k] - b[1][k]]], np.int32)
    got, iou = api.hog_box_windows(W, H, box, [s], (fw, fh), cell, 9, 1, pad=(px, py))
    ref, _ = T.box_windows(W, H, box, [((lw, lh), (31, hh, hw))], cell, fw, fh, px, py, 0.5)
    assert got[0].tolist() == [0, 3, 2] and iou[0] == 1.0
    assert np.array_equal(got, ref)


@pytest.mark.parametrize("N,D,lam", [(60, 5, 0.1), (200, 12, 1.0), (150, 30, 0.01), (40, 60, 0.5)])
def test_newton_reference_reaches_the_optimum(N, D, lam):
    rng = np.random.default_rng(N + D)
    A = rng.standard_normal((N, D))
    A[:, -1] = 1.0
    y = np.where(A[:, :-1] @ rng.standard_normal(D - 1) + 0.3 * rng.standard_normal(N) > 0, 1.0, -1.0)
    w, its, act = T.svm_newton(A, y, lam)
    res = so.minimize(lambda v: T.svm_objective(A, y, lam, v), np.zeros(D), jac=lambda v: T.svm_gradient(A, y, lam, v),
                      method="L-BFGS-B", options={"gtol": 1e-12, "ftol": 1e-15, "maxiter": 10000})
    f, f_ref = T.svm_objective(A, y, lam, w), float(res.fun)
    g = T.svm_gradient(A, y, lam, w)
    print(f"N {N} D {D}: {its} Newton steps, |S| {act.size}, f {f:.12g} (scipy {f_ref:.12g}), |grad| {np.abs(g).max():.2e}")
    assert f <= f_ref + 1e-9 * max(1.0, abs(f_ref))
    assert np.abs(g).max() <= 1e-8 * max(1.0, np.abs(A).max() * np.sqrt(N))
    # at the optimum the Newton point is the ridge solution on its own active set
    assert np.allclose(w, T.ridge_on(A, y, lam, act), rtol=1e-9, atol=1e-10)


def test_box_windows_refusals():
    ok = dict(width=100, height=80, boxes=[[10, 10, 30, 30]], scales=[1.0], filter_size=(4, 4), cell_size=8, num_bins=9)
    api.hog_box_windows(**ok)
    bad = [dict(width=0), dict(height=0), dict(scales=[]), dict(scales=[0.0]), dict(scales=[5.0]), dict(scales=[float("nan")]),
           dict(cell_size=0), dict(cell_size=33), dict(num_bins=0), dict(num_bins=17), dict(variant=2), dict(filter_size=(0, 4)),
           dict(filter_size=(33, 4)), dict(pad=(4, 0)), dict(pad=(0, -1)), dict(positive_overlap=1.5),
           dict(positive_overlap=-0.1), dict(boxes=[[0, 0, 0, 5]]), dict(boxes=[[0, 0, 5, -1]])]
    for b in bad:
        with pytest.raises(SdError):
            api.hog_box_windows(**{**ok, **b})

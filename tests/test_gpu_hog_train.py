"""Training HOG filters on the device: sd_hog_windows, sd_learn_squared_hinge and sd_hog_train_filter (api.vl_hog_windows,
api.learn_squared_hinge, api.train_hog_filter).

- Window rows are numpy slicing of the maps bit for bit, with pads, flips and grids of different sizes; canaries around the rows
  and in the ldr gap survive; a flipped row is the unflipped row of the mirrored position in vl_hog_flip's grid; row . [F | b]
  in float64 is vl_hog_correlate's score within the float32 bound of its FMA chain; every refusal writes nothing.
- The SVM's w is within tests/chol_ref.py's per-element bars of the float64 ridge solution on its final active set, at D <= 256
  (the LU route) and D > 256 (the centred Cholesky), on random rows and on HOG rows from the gather; every row's float64 margin
  agrees with that set except rows within the margin bar of 1; f decreases at every step.
- The trainer's filter and bias are learn_squared_hinge on the rows rebuilt from its negatives and the assigned positives with
  the public primitives, bit for bit; two runs are identical.
- Trained on 48 seeded planted-object frames, vl_hog_detect reaches VOC AP >= 0.9 on 32 held-out frames, no lower than with
  rounds = 0, and the training frames' false positives above score 0 do not rise from round to round.
- Trained on the five golden example frames, each face is its frame's top detection at IoU >= 0.5 and goes on to landmarks."""
import numpy as np
import pytest
import torch

import chol_ref as CR
import hog_train_ref as T
from superviseddescent_b200 import _capi
from superviseddescent_b200._capi import SdError

pytestmark = pytest.mark.gpu

CANARY = np.float32(-1234.5)
U = 2.0 ** -24


def _maps(rng, sizes, dd):
    return [torch.from_numpy(rng.uniform(0, 0.4, (dd, h, w)).astype(np.float32)).cuda() for h, w in sizes]


def _window_ref(m, x, y, fw, fh, px, py):
    dd, h, w = m.shape
    pad = np.zeros((dd, h + 2 * fh, w + 2 * fw), np.float32)
    pad[:, fh:fh + h, fw:fw + w] = m
    return pad[:, fh + y - py:fh + y - py + fh, fw + x - px:fw + x - px + fw]


def _random_windows(rng, sizes, fw, fh, px, py, n):
    out = []
    for _ in range(n):
        g = int(rng.integers(0, len(sizes)))
        h, w = sizes[g]
        oh, ow = h + 2 * py - fh + 1, w + 2 * px - fw + 1
        if oh > 0 and ow > 0:
            out.append((g, int(rng.integers(0, ow)), int(rng.integers(0, oh)), int(rng.integers(0, 2))))
    return np.asarray(out, np.int32)


@pytest.mark.parametrize("K,variant,fw,fh,px,py", [(9, 1, 6, 6, 0, 0), (4, 0, 5, 3, 2, 1), (16, 1, 3, 7, 1, 6), (2, 1, 1, 1, 0, 0)])
def test_windows_are_slices_of_the_maps(sd, K, variant, fw, fh, px, py):
    rng = np.random.default_rng(K * 100 + fw)
    dd = sd._hog_dims(K, variant)
    sizes = [(9, 13), (fh, fw), (20, 7), (3, 30), (1, 1)]
    maps = _maps(rng, sizes, dd)
    win = _random_windows(rng, sizes, fw, fh, px, py, 300)
    D = dd * fw * fh + 1
    ldr = D + 5
    rows = torch.full((len(win) + 2, ldr), float(CANARY), device="cuda")
    g, keep = sd._maps_table(maps, dd, "cuda")
    d_w = torch.from_numpy(win).cuda()
    ctx = sd.default_context()
    rc = _capi.lib().sd_hog_windows(ctx.h, sd.C.byref(g), K, variant, fw, fh, px, py, _capi.ptr(d_w), len(win),
                                    _capi.ptr(rows[1:]), ldr)
    assert rc == 0
    got = rows.cpu().numpy()
    perm = sd.vl_hog_permutation(variant, K)
    for r, (gi, x, y, fl) in enumerate(win):
        blk = _window_ref(maps[gi].cpu().numpy(), x, y, fw, fh, px, py)
        if fl:
            blk = blk[perm][:, :, ::-1]
        ref = np.concatenate([blk.ravel(), [1.0]]).astype(np.float32)
        assert np.array_equal(got[1 + r, :D].view(np.uint32), ref.view(np.uint32)), (r, gi, x, y, fl)
    assert (got[0] == CANARY).all() and (got[-1] == CANARY).all() and (got[1:-1, D:] == CANARY).all()
    # the public wrapper gives the same rows
    assert torch.equal(sd.vl_hog_windows(maps, win, (fw, fh), K, variant, pad=(px, py)), rows[1:-1, :D])


def test_flip_identity_through_relayout(sd):
    rng = np.random.default_rng(5)
    K, variant, fw, fh, px, py = 9, 1, 5, 4, 2, 1
    dd = sd._hog_dims(K, variant)
    sizes = [(11, 17), (6, 9)]
    maps = _maps(rng, sizes, dd)
    flipped = sd.vl_hog_flip(maps, K, variant)
    win = _random_windows(rng, sizes, fw, fh, px, py, 200)
    win[:, 3] = 1
    a = sd.vl_hog_windows(maps, win, (fw, fh), K, variant, pad=(px, py))
    mirror = win.copy()
    for r, (gi, x, y, _) in enumerate(win):
        ow = sizes[gi][1] + 2 * px - fw + 1
        mirror[r] = (gi, ow - 1 - x, y, 0)
    b = sd.vl_hog_windows(flipped, mirror, (fw, fh), K, variant, pad=(px, py))
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_row_dot_filter_is_the_score(sd):
    rng = np.random.default_rng(9)
    K, variant, fw, fh, px, py = 9, 1, 6, 5, 3, 2
    dd = sd._hog_dims(K, variant)
    sizes = [(14, 19), (8, 8)]
    maps = _maps(rng, sizes, dd)
    F = torch.from_numpy(rng.standard_normal((1, dd, fh, fw)).astype(np.float32)).cuda()
    b = np.float32(0.37)
    scores = sd.vl_hog_correlate(maps, F, K, variant, bias=[b], pad=(px, py))
    worst = 0.0
    for gi, (h, w) in enumerate(sizes):
        oh, ow = h + 2 * py - fh + 1, w + 2 * px - fw + 1
        yy, xx = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
        win = np.stack([np.full(xx.size, gi), xx.ravel(), yy.ravel(), np.zeros(xx.size)], 1).astype(np.int32)
        rows = sd.vl_hog_windows(maps, win, (fw, fh), K, variant, pad=(px, py)).cpu().numpy().astype(np.float64)
        fb = np.concatenate([F.cpu().numpy().ravel(), [b]]).astype(np.float64)
        exact = rows @ fb
        n = fb.size
        bar = (n * U / (1 - n * U)) * (np.abs(rows) @ np.abs(fb)) + U * np.abs(exact)   # the FMA chain and the bias add
        got = scores[gi][0].cpu().numpy().ravel().astype(np.float64)
        worst = max(worst, float(np.max(np.abs(got - exact) / bar)))
    print(f"score vs row . [F | b]: worst error / bar {worst:.4f}")
    assert worst <= 1.0


def test_window_refusals_write_nothing(sd):
    rng = np.random.default_rng(2)
    K, variant, fw, fh = 9, 1, 4, 4
    dd = sd._hog_dims(K, variant)
    sizes = [(6, 8), (5, 5)]
    maps = _maps(rng, sizes, dd)
    D = dd * fw * fh + 1
    g, keep = sd._maps_table(maps, dd, "cuda")
    ctx = sd.default_context()
    good = np.asarray([[0, 1, 1, 0], [1, 0, 0, 1]], np.int32)
    cases = [  # (windows, K, variant, fw, fh, px, py, ldr)
        (np.asarray([[2, 0, 0, 0]], np.int32), K, variant, fw, fh, 0, 0, D),
        (np.asarray([[-1, 0, 0, 0]], np.int32), K, variant, fw, fh, 0, 0, D),
        (np.asarray([[0, 5, 0, 0]], np.int32), K, variant, fw, fh, 0, 0, D),          # ow = 5
        (np.asarray([[0, 0, 3, 0]], np.int32), K, variant, fw, fh, 0, 0, D),          # oh = 3
        (np.asarray([[1, 0, 0, 0]], np.int32), K, variant, fw, fh, 0, 0, D),          # grid 1 is 5 x 5: ok
        (np.asarray([[1, 2, 0, 0]], np.int32), K, variant, fw, fh, 0, 0, D),          # ow = 2
        (np.asarray([[0, 0, 0, 2]], np.int32), K, variant, fw, fh, 0, 0, D),
        (np.asarray([[0, 0, 0, -1]], np.int32), K, variant, fw, fh, 0, 0, D),
        (good, K, variant, fw, fh, 0, 0, D - 1),
        (good, K, variant, fw, fh, 4, 0, D),
        (good, K, variant, 33, fh, 0, 0, 33 * fh * dd + 1),
        (good, 17, variant, fw, fh, 0, 0, D),
        (good, K, 2, fw, fh, 0, 0, D),
    ]
    for i, (w, k, v, a, b, px, py, ldr) in enumerate(cases):
        rows = torch.full((4, max(ldr, 1)), float(CANARY), device="cuda")
        d_w = torch.from_numpy(w).cuda()
        rc = _capi.lib().sd_hog_windows(ctx.h, sd.C.byref(g), k, v, a, b, px, py, _capi.ptr(d_w), len(w), _capi.ptr(rows), ldr)
        torch.cuda.synchronize()
        if i == 4:
            assert rc == 0
            continue
        assert rc == 1, i
        assert (rows.cpu().numpy() == CANARY).all(), i
    rows = torch.full((4, D), float(CANARY), device="cuda")
    d_w = torch.from_numpy(good).cuda()
    rc = _capi.lib().sd_hog_windows(ctx.h, sd.C.byref(g), K, variant, fw, fh, 0, 0, _capi.ptr(d_w).value + 2, 1, _capi.ptr(rows), D)
    assert rc == 1 and (rows.cpu().numpy() == CANARY).all()


# ---- the SVM -----------------------------------------------------------------------------------------------------------------
def _svm_problem(rng, N, D, hog_like):
    if hog_like:
        A = rng.gamma(2.0, 0.05, (N, D)).astype(np.float32)
    else:
        A = rng.standard_normal((N, D)).astype(np.float32)
    A[:, -1] = 1.0
    u = rng.standard_normal(D - 1)
    s = (A[:, :-1].astype(np.float64) - A[:, :-1].mean(0)) @ u
    y = np.where(s + 0.5 * s.std() * rng.standard_normal(N) > 0, 1.0, -1.0).astype(np.float32)
    return A, y


def _check_svm(sd, A, y, lam, name):
    N, D = A.shape
    w, rep = sd.learn_squared_hinge(A, y, lam, max_iterations=100)
    w = w.cpu().numpy()
    assert rep.stop == "converged", rep
    # the final active set as an input: the float64 ridge solution on it, with chol_ref's bars
    o = A.astype(np.float64) @ w.astype(np.float64)
    act = np.flatnonzero(y * o < 1)
    assert act.size == rep.active
    mu, Ac = CR.centre_restated(A[act], False)
    if D > CR.LU_MAX_DIM:
        mu, _ = CR.centre_restated(A, False)                      # the shift of the whole solve: the means of all rows
        Ac = (A[act] - mu).astype(np.float32)
    tr = CR.learn_truth(Ac, y[act, None], lam, False)
    bw = tr.bar_w(0)
    r = CR.ratio(w[:-1, None], tr.w, bw)
    x_true = tr.xb - mu[:-1].astype(np.float64) @ tr.w
    bxb = tr.bar_xb(bw) + np.abs(mu[:-1].astype(np.float64)) @ bw + 2 * U * np.abs(x_true)
    rb = float(np.max(np.abs(w[-1] - x_true) / bxb))
    # margins: membership agrees with the float64 margin of the true solution except within the margin bar of 1
    wt = np.concatenate([tr.w[:, 0], x_true])
    o_true = A.astype(np.float64) @ wt
    mbar = np.abs(A[:, :-1].astype(np.float64)) @ bw[:, 0] + bxb[0] + 1e-12
    disagree = (y * o_true < 1) != (y * o < 1)
    near = np.abs(y * o_true - 1) <= mbar
    print(f"{name}: N {N} D {D}, {rep.iterations} steps, |S| {rep.active}, f {rep.objective:.6g}, error / bar {r.max():.4f} "
          f"(bias {rb:.4f}), {int(disagree.sum())} memberships differ, {int(near.sum())} rows within the margin bar")
    assert r.max() <= 1.0 and rb <= 1.0
    assert not (disagree & ~near).any()
    # f decreases at every step: the run capped at k steps is the prefix of the full run
    fs = [sd.learn_squared_hinge(A, y, lam, max_iterations=k)[1].objective for k in range(1, rep.iterations + 1)]
    assert all(b < a for a, b in zip(fs, fs[1:])), fs
    assert fs[-1] == rep.objective
    return w, rep


@pytest.mark.parametrize("N,D,lam,hog_like", [(400, 40, 0.5, False), (900, 200, 2.0, True), (1500, 300, 1.0, True),
                                              (2000, 513, 4.0, True)])
def test_svm_within_the_bars_of_its_active_set(sd, N, D, lam, hog_like):
    A, y = _svm_problem(np.random.default_rng(N + D), N, D, hog_like)
    _check_svm(sd, A, y, lam, "random" if not hog_like else "hog-like")


def test_svm_on_gathered_hog_rows(sd):
    frames, boxes = T.planted_frames(3, 6, 320, 240, sides=(48, 96))
    cell, K, fw, fh = 8, 9, 4, 4                           # D = 31 * 16 + 1 = 497: the centred Cholesky
    scales = T.detector_scales(320, 240, cell, fw)
    feats, _ = sd.vl_hog_pyramid(frames, scales, cell, K, 1)
    maps = [m for row in feats for m in row if m is not None and m.shape[1] >= fh and m.shape[2] >= fw]
    rng = np.random.default_rng(4)
    sizes = [tuple(m.shape[1:]) for m in maps]
    win = _random_windows(rng, sizes, fw, fh, 0, 0, 1200)
    A = sd.vl_hog_windows(maps, win, (fw, fh), K, 1).cpu().numpy()
    y = np.where(win[:, 3] == 1, 1.0, -1.0).astype(np.float32)     # mirrored windows against the others
    _check_svm(sd, A, y, 0.5, "gathered rows")


def test_svm_refusals_write_nothing(sd):
    A, y = _svm_problem(np.random.default_rng(0), 50, 8, False)
    ctx = sd.default_context()
    dA, dy = torch.from_numpy(A).cuda(), torch.from_numpy(y).cuda()
    bad_y = dy.clone()
    bad_y[7] = 0.5
    cases = [(dA, 8, dy, 50, 8, 1.0, 10), (dA, 8, bad_y, 50, 8, 1.0, 10), (dA, 8, dy, 50, 8, 0.0, 10), (dA, 8, dy, 50, 8, -1.0, 10),
             (dA, 8, dy, 0, 8, 1.0, 10), (dA, 8, dy, 50, 1, 1.0, 10), (dA, 8, dy, 50, 8, 1.0, 0), (dA, 7, dy, 50, 8, 1.0, 10),
             (dA, 8, dy, 50, 8, float("nan"), 10)]
    for i, (a, lda, yy, N, D, lam, it) in enumerate(cases):
        w = torch.full((8,), float(CANARY), device="cuda")
        rc = _capi.lib().sd_learn_squared_hinge(ctx.h, _capi.ptr(a), lda, _capi.ptr(yy), N, D, lam, it, _capi.ptr(w), None)
        torch.cuda.synchronize()
        if i == 0:
            assert rc == 0
            continue
        assert rc == 1, i
        assert (w.cpu().numpy() == CANARY).all(), i


# ---- the trainer ---------------------------------------------------------------------------------------------------------------
CELL, K, SIDE = 8, 9, 6


def _train(sd, frames, boxes, scales, **kw):
    p = dict(lam=0.01, rounds=3, negatives_per_frame=16, max_negatives=4000, flip_positives=True)
    p.update(kw)
    return sd.train_hog_filter(frames, np.arange(len(boxes)), boxes, scales, (SIDE, SIDE), CELL, K, **p)


def test_trainer_is_the_svm_on_its_rows_and_deterministic(sd):
    frames, boxes = T.planted_frames(21, 10, 320, 240, sides=(48, 120))
    scales = T.detector_scales(320, 240, CELL, SIDE)
    hf = _train(sd, frames, boxes, scales, rounds=2, max_negatives=300)
    hf2 = _train(sd, frames, boxes, scales, rounds=2, max_negatives=300)
    assert torch.equal(hf.filter.view(torch.int32), hf2.filter.view(torch.int32)) and hf.bias == hf2.bias
    assert np.array_equal(hf.negatives, hf2.negatives)
    assert [{k: r[k] for k in T.COUNTS + ("solve",)} for r in hf.report] == [{k: r[k] for k in T.COUNTS + ("solve",)} for r in hf2.report]
    for r in hf.report:
        print(r)
    # rebuild the rows: the assigned positives (box order, each followed by its mirror), then the cache in slot order
    feats, _ = sd.vl_hog_pyramid(frames, scales, CELL, K, 1)
    S = len(scales)
    maps, index = [], {}
    for f in range(len(frames)):
        for s in range(S):
            if feats[f][s] is not None:
                index[(f, s)] = len(maps)
                maps.append(feats[f][s])
    win = []
    for f, b in enumerate(boxes):
        lv, iou = sd.hog_box_windows(320, 240, b[None], scales, (SIDE, SIDE), CELL, K)
        if lv[0, 0] >= 0:
            win += [(index[(f, lv[0, 0])], lv[0, 1], lv[0, 2], 0), (index[(f, lv[0, 0])], lv[0, 1], lv[0, 2], 1)]
    npos = len(win)
    win += [(index[(f, s)], x, y, 0) for f, s, x, y in hf.negatives]
    A = sd.vl_hog_windows(maps, np.asarray(win, np.int32), (SIDE, SIDE), K, 1)
    y = torch.tensor([1.0] * npos + [-1.0] * (len(win) - npos), device="cuda")
    w, rep = sd.learn_squared_hinge(A, y, 0.01, max_iterations=50)
    last = [r for r in hf.report if r["solve"] is not None][-1]
    assert rep == last["solve"]
    assert torch.equal(w[:-1].view(torch.int32), hf.filter.reshape(-1).view(torch.int32))
    assert w[-1].item() == hf.bias


def test_trainer_follows_the_rule(sd):
    # a cache small enough that round 0 truncates and later rounds evict inactive negatives
    frames, boxes = T.planted_frames(77, 10, 240, 180, sides=(48, 96), distractors=5)
    scales = T.detector_scales(240, 180, CELL, 5)
    box_frame = np.asarray([0, 1, 2, 3, 4, 5, 6, 7], np.int64)        # frames 8 and 9 are pure negative frames
    kw = dict(lam=0.1, flip_positives=True, rounds=4, negatives_per_frame=16, mine_overlap=0.5, max_negatives=40,
              negative_overlap=0.3, positive_overlap=0.6, max_iterations=50)
    hf = sd.train_hog_filter(frames, box_frame, boxes[:8], scales, (5, 5), CELL, K, **kw)
    filt, bias, neg, reps = T.train_rule(sd, frames, box_frame, boxes[:8], scales, (5, 5), CELL, K, **kw)
    for r in hf.report:
        print({k: r[k] for k in T.COUNTS + ("solve",)})
    assert np.array_equal(hf.negatives, neg)
    got = [{k: r[k] for k in T.COUNTS + ("solve",)} for r in hf.report]
    assert got[:len(reps)] == reps
    assert all(r["solved"] == 0 and r["positives"] == 0 for r in got[len(reps):])      # zero after an early stop
    assert np.array_equal(hf.filter.cpu().numpy().ravel().view(np.uint32), filt.view(np.uint32))
    assert np.float32(hf.bias) == bias
    assert sum(r["truncated"] for r in reps) > 0 and sum(r["evicted"] for r in reps) > 0
    assert sum(r["excluded"] for r in reps) > 0
    # the phase timings are filled in for every round that ran
    assert all(r["times_ms"]["pyramid"] > 0 and r["times_ms"]["gather"] > 0 for r in hf.report[:len(reps)] if r["added"])


def test_svm_with_one_class(sd):
    # every label +1: the optimum is w' = 0 with bias 1, where the active set may be empty
    rng = np.random.default_rng(3)
    A = rng.standard_normal((200, 20)).astype(np.float32)
    A[:, -1] = 1.0
    for y in (np.ones(200, np.float32), -np.ones(200, np.float32)):
        w, rep = sd.learn_squared_hinge(A, y, 1.0)
        w = w.cpu().numpy()
        print(rep, np.abs(w[:-1]).max(), w[-1])
        assert rep.stop in ("converged", "no decrease")
        assert np.abs(w[:-1]).max() <= 1e-5 and abs(w[-1] - y[0]) <= 1e-5
        assert rep.objective <= 1e-8


def _detect_fp(sd, frames, boxes, scales, hf, thr):
    d = sd.vl_hog_detect(frames, scales, hf.filter[None], CELL, K, threshold=thr, bias=[hf.bias], overlap=0.3, max_detections=64)
    return d


def _ap(sd, frames, boxes, scales, hf):
    d = _detect_fp(sd, frames, boxes, scales, hf, -2.0)
    return T.voc_ap(d.frame, d.boxes, d.scores, boxes)


def _false_positives(sd, frames, boxes, scales, hf):
    d = _detect_fp(sd, frames, boxes, scales, hf, 0.0)
    fp = 0
    for f, (x, y, w, h) in zip(d.frame, d.boxes):
        gx, gy, gw, gh = boxes[f]
        iw = max(0, min(x + w, gx + gw) - max(x, gx))
        ih = max(0, min(y + h, gy + gh) - max(y, gy))
        fp += iw * ih < 0.5 * (w * h + gw * gh - iw * ih)
    return int(fp)


def test_trained_detector_quality(sd):
    W, H = 320, 240
    frames, boxes = T.planted_frames(1234, 80, W, H, sides=(48, 120))
    train, test = slice(0, 48), slice(48, 80)
    scales = T.detector_scales(W, H, CELL, SIDE)
    fps, aps = [], []
    for rounds in range(0, 4):
        hf = _train(sd, frames[train], boxes[train], scales, rounds=rounds)
        aps.append(_ap(sd, frames[test], boxes[test], scales, hf))
        fps.append(_false_positives(sd, frames[train], boxes[train], scales, hf))
    print(f"held-out AP by rounds 0..3: {[round(a, 4) for a in aps]}; training false positives above 0: {fps}")
    assert aps[-1] >= 0.9
    assert aps[-1] >= aps[0]
    assert all(b <= a for a, b in zip(fps, fps[1:])), fps


def test_golden_faces_train_and_chain_to_landmarks(sd, golden):
    ex = golden.examples
    grays = [np.ascontiguousarray(ex[f"gray{i}"]) for i in range(5)]
    boxes = np.asarray(ex["boxes"][:5], np.int32)
    side = 8
    sides = [int(b[2]) for b in boxes]
    s_hi, s_lo = side * CELL * 1.3 / min(sides), side * CELL * 0.7 / max(sides)
    scales = [s_hi * (s_lo / s_hi) ** (k / 11) for k in range(12)]
    hf = sd.train_hog_filter(grays, np.arange(5), boxes, scales, (side, side), CELL, K, lam=0.01, flip_positives=True, rounds=3,
                             negatives_per_frame=64, max_negatives=4000)
    d = sd.vl_hog_detect(grays, scales, hf.filter[None], CELL, K, threshold=-10.0, bias=[hf.bias], overlap=0.3, max_detections=8)
    model = sd.load_detection_model(golden.model_path)
    for i in range(5):
        k = int(np.flatnonzero(d.frame == i)[0])
        x, y, w, h = (int(v) for v in d.boxes[k])
        bx, by, bw, bh = (int(v) for v in boxes[i])
        iw = max(0, min(x + w, bx + bw) - max(x, bx))
        ih = max(0, min(y + h, by + bh) - max(y, by))
        iou = iw * ih / (w * h + bw * bh - iw * ih)
        print(f"face {i}: top detection {d.boxes[k].tolist()} score {d.scores[k]:.3f}, golden {boxes[i].tolist()}, IoU {iou:.3f}")
        assert iou >= 0.5
        lm = model.detect_faces([grays[i]], np.zeros(1, np.int32), boxes=d.boxes[k:k + 1])
        assert np.isfinite(lm).all()


def test_trainer_refusals(sd):
    frames, boxes = T.planted_frames(5, 2, 160, 120, sides=(48, 60))
    scales = [1.0, 0.8]
    _train(sd, frames, boxes, scales, rounds=0)
    bad = [dict(lam=0.0), dict(positive_overlap=1.5), dict(negative_overlap=-0.1), dict(mine_overlap=2.0), dict(rounds=-1),
           dict(negatives_per_frame=0), dict(negatives_per_frame=8193), dict(max_negatives=0), dict(max_iterations=0),
           dict(positive_overlap=1.0)]                                  # no window covers a box exactly: nothing to train on
    for b in bad:
        with pytest.raises((SdError, ValueError)):
            _train(sd, frames, boxes, scales, **b)
    with pytest.raises(SdError):
        sd.train_hog_filter(frames, [0, 5], boxes, scales, (SIDE, SIDE), CELL, K)       # a box of a missing frame
    with pytest.raises(SdError):
        sd.train_hog_filter(frames, [0, 1], boxes, scales, (17, 17), CELL, 16, 0)       # D = 64 * 289 + 1 > SD_HOG_TRAIN_MAX_DIM

"""Oracles of the HOG filter trainer (include/sd_b200.h: sd_hog_box_windows, sd_learn_squared_hinge, sd_hog_train_filter), the
seeded planted-object generator that the tests and bench_hog_train.py share, and VOC average precision.

- `box_windows` restates sd_hog_box_windows: every score position of every non-empty level, its box by hog_detect_ref's integer
  rule, the IoU as an exact Fraction, ties to the lower level, then y, then x.
- `svm_newton` is the primal finite Newton method in float64 with the exact line search; `svm_objective` and `svm_gradient` are
  f and its gradient, for the KKT check.
- `planted_frames` draws grey frames with one planted object each (a ringed, crossed square at sides in a range) and textured
  distractors of the same size range, from a seed.
"""
from fractions import Fraction

import numpy as np

import hog_detect_ref as DR


class _Level:
    def __init__(self, frame_w, frame_h, level_w, level_h):
        self.frame_w, self.frame_h, self.level_w, self.level_h = frame_w, frame_h, level_w, level_h


def box_windows(frame_w, frame_h, boxes, levels, cell, fw, fh, pad_x, pad_y, positive_overlap):
    """levels: per scale ((level_w, level_h), (dd, hog_h, hog_w)) as api.hog_pyramid_shape gives them.  -> (n, 3) int32 of
    (level, x, y) (level -1: unassigned) and (n,) float64 IoU."""
    cands = []                                        # (level, y, x, x0, y0, x1, y1), in tie order
    for s, ((lw, lh), (_, hh, hw)) in enumerate(levels):
        if hw == 0:
            continue
        oh, ow = hh + 2 * pad_y - fh + 1, hw + 2 * pad_x - fw + 1
        if oh <= 0 or ow <= 0:
            continue
        yy, xx = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
        b = DR.boxes(xx.ravel(), yy.ravel(), _Level(frame_w, frame_h, lw, lh), cell, fw, fh, pad_x, pad_y)
        cands.append((np.full(oh * ow, s), yy.ravel(), xx.ravel()) + tuple(b))
    out = np.full((len(boxes), 3), 0, np.int32)
    out[:, 0] = -1
    iou = np.zeros(len(boxes))
    if not cands:
        return out, iou
    lv, yy, xx, x0, y0, x1, y1 = (np.concatenate([c[k] for c in cands]) for k in range(7))
    for i, (bx, by, bw, bh) in enumerate(np.asarray(boxes, np.int64)):
        iw = np.minimum(x1, bx + bw) - np.maximum(x0, bx)
        ih = np.minimum(y1, by + bh) - np.maximum(y0, by)
        inter = np.where((iw > 0) & (ih > 0), iw * ih, 0)
        union = (x1 - x0) * (y1 - y0) + bw * bh - inter
        best, arg = None, -1
        # a float pre-filter, then exact rationals among the near-best
        r = inter / union
        for k in np.flatnonzero(r >= r.max() * (1 - 1e-9)):
            v = Fraction(int(inter[k]), int(union[k]))
            if best is None or v > best:             # candidates are in tie order: the first of equals stays
                best, arg = v, k
        iou[i] = float(inter[arg]) / float(union[arg])
        if float(inter[arg]) >= positive_overlap * float(union[arg]):
            out[i] = (lv[arg], xx[arg], yy[arg])
    return out, iou


# ---- the squared-hinge SVM -----------------------------------------------------------------------------------------------
def svm_objective(A, y, lam, w):
    A = np.asarray(A, np.float64)
    w = np.asarray(w, np.float64)
    r = np.maximum(0.0, 1.0 - y * (A @ w))
    return 0.5 * lam * float(w[:-1] @ w[:-1]) + 0.5 * float(r @ r)


def svm_gradient(A, y, lam, w):
    A = np.asarray(A, np.float64)
    w = np.asarray(w, np.float64)
    r = np.maximum(0.0, 1.0 - y * (A @ w))
    g = -A.T @ (y * r)
    g[:-1] += lam * w[:-1]
    return g


def ridge_on(A, y, lam, rows):
    """(lam I' + A_S^T A_S) w = A_S^T y_S in float64 on the rows `rows`, the bias (last column) unregularised"""
    A = np.asarray(A, np.float64)[rows]
    D = A.shape[1]
    H = A.T @ A
    H[np.arange(D - 1), np.arange(D - 1)] += lam
    return np.linalg.solve(H, A.T @ np.asarray(y, np.float64)[rows])


def _line_search(A, y, lam, w, d):
    o, dl = A @ w, A @ d
    al, be = 1.0 - y * o, y * dl
    a, b = lam * float(d[:-1] @ d[:-1]), lam * float(w[:-1] @ d[:-1])
    act = (al > 0) | ((al == 0) & (be < 0))
    a += float(be[act] @ be[act])
    b -= float(be[act] @ al[act])
    brk = sorted([(al[i] / be[i], i) for i in np.flatnonzero((act & (be > 0)) | (~act & (be < 0)))])
    t0 = 0.0
    for t, i in brk:
        if a > 0 and -b / a <= t:
            return max(t0, -b / a)
        sgn = -1.0 if be[i] > 0 else 1.0
        a += sgn * be[i] ** 2
        b -= sgn * be[i] * al[i]
        t0 = t
    return max(t0, -b / a) if a > 0 else 1.0


def svm_newton(A, y, lam, max_iterations=100):
    """-> (w, iterations, final active rows): the primal finite Newton method of sd_learn_squared_hinge in float64"""
    A = np.asarray(A, np.float64)
    y = np.asarray(y, np.float64)
    w = np.zeros(A.shape[1])
    act = np.arange(A.shape[0])
    f = svm_objective(A, y, lam, w)
    for it in range(1, max_iterations + 1):
        wn = ridge_on(A, y, lam, act)
        act_n = np.flatnonzero(y * (A @ wn) < 1)
        if not np.array_equal(act_n, act):
            t = _line_search(A, y, lam, w, wn - w)
            wn = w + t * (wn - w)
            act_n = np.flatnonzero(y * (A @ wn) < 1)
        fn = svm_objective(A, y, lam, wn)
        if not fn < f:
            return w, it, act
        same = np.array_equal(act_n, act)
        w, f, act = wn, fn, act_n
        if same:
            return w, it, act
    return w, max_iterations, act


# ---- the planted-object generator ------------------------------------------------------------------------------------------
def _object(side, rng):
    """a bright ringed square with a dark cross, side x side pixels, with a little intensity jitter"""
    t = np.linspace(-1, 1, side)
    X, Y = np.meshgrid(t, t)
    r = np.maximum(np.abs(X), np.abs(Y))
    img = np.where(r > 0.78, 220.0, 110.0)
    img = np.where((np.abs(X - Y) < 0.16) | (np.abs(X + Y) < 0.16), 30.0, img)
    img = np.where(r > 0.97, 60.0, img)
    return img + rng.normal(0, 6, img.shape)


def _distractor(side, rng):
    kind = rng.integers(0, 3)
    if kind == 0:                                         # blocky noise
        k = max(2, side // int(rng.integers(4, 12)))
        small = rng.uniform(20, 235, (side // k + 1, side // k + 1))
        return np.kron(small, np.ones((k, k)))[:side, :side]
    t = np.linspace(-1, 1, side)
    X, Y = np.meshgrid(t, t)
    if kind == 1:                                         # concentric circles
        return 128 + 90 * np.sin(float(rng.uniform(6, 14)) * np.sqrt(X * X + Y * Y))
    a = float(rng.uniform(0, np.pi))                      # oriented stripes
    return 128 + 100 * np.sign(np.sin(float(rng.uniform(5, 12)) * (np.cos(a) * X + np.sin(a) * Y)))


def planted_frames(seed, n, width, height, sides=(48, 160), distractors=4):
    """-> (frames (n, height, width) uint8, boxes (n, 4) int32: the planted object's (x, y, side, side) per frame)"""
    rng = np.random.default_rng(seed)
    frames = np.empty((n, height, width), np.uint8)
    boxes = np.zeros((n, 4), np.int32)
    for i in range(n):
        img = rng.normal(128, 12, (height // 8 + 1, width // 8 + 1))
        img = np.kron(img, np.ones((8, 8)))[:height, :width] + rng.normal(0, 4, (height, width))
        placed = []

        def place(side):
            for _ in range(50):
                x, y = int(rng.integers(0, width - side)), int(rng.integers(0, height - side))
                if all(x + side <= px or px + ps <= x or y + side <= py or py + ps <= y for px, py, ps in placed):
                    placed.append((x, y, side))
                    return x, y
            return None

        side = int(rng.integers(sides[0], min(sides[1], height - 1, width - 1) + 1))
        x, y = place(side)
        img[y:y + side, x:x + side] = _object(side, rng)
        boxes[i] = (x, y, side, side)
        for _ in range(distractors):
            s = int(rng.integers(sides[0], min(sides[1], height - 1, width - 1) + 1))
            at = place(s)
            if at:
                img[at[1]:at[1] + s, at[0]:at[0] + s] = _distractor(s, rng)
        frames[i] = np.clip(img, 0, 255).astype(np.uint8)
    return frames, boxes


def detector_scales(width, height, cell, side_cells, step=5):
    """2^(-l / step) while a level still holds a side_cells x side_cells-cell filter"""
    out, l = [], 0
    while min(width, height) * 2.0 ** (-l / step) >= cell * (side_cells + 1):
        out.append(2.0 ** (-l / step))
        l += 1
    return out


def voc_ap(frame, boxes, scores, gt, iou_min=0.5):
    """VOC all-point average precision of detections (frame (n,), boxes (n, 4) x y w h, scores (n,)) against one ground-truth box
    per frame, gt (F, 4); each ground truth is matched at most once, by detections in score order"""
    order = np.argsort(-np.asarray(scores, np.float64), kind="stable")
    used = np.zeros(len(gt), bool)
    tp = np.zeros(len(order))
    for k, j in enumerate(order):
        f = int(frame[j])
        x, y, w, h = (int(v) for v in boxes[j])
        gx, gy, gw, gh = (int(v) for v in gt[f])
        iw = max(0, min(x + w, gx + gw) - max(x, gx))
        ih = max(0, min(y + h, gy + gh) - max(y, gy))
        inter = iw * ih
        if not used[f] and inter >= iou_min * (w * h + gw * gh - inter):
            used[f] = True
            tp[k] = 1
    ctp = np.cumsum(tp)
    rec = ctp / len(gt)
    prec = ctp / np.arange(1, len(order) + 1)
    mrec = np.concatenate([[0.0], rec, [1.0]])
    mpre = np.concatenate([[0.0], prec, [0.0]])
    for i in range(len(mpre) - 2, -1, -1):
        mpre[i] = max(mpre[i], mpre[i + 1])
    idx = np.flatnonzero(mrec[1:] != mrec[:-1])
    return float(np.sum((mrec[idx + 1] - mrec[idx]) * mpre[idx + 1]))


# ---- the trainer's rule (include/sd_b200.h, sd_hog_train_filter) on the public primitives ------------------------------------
COUNTS = ("positives", "unassigned", "cache", "mined", "excluded", "added", "evicted", "truncated", "solved")


def _iou_exceeds(a, b, overlap):
    """(double) inter > overlap * (double) union for boxes (x, y, w, h) in int64 pixel areas"""
    iw = min(a[0] + a[2], b[0] + b[2]) - max(a[0], b[0])
    ih = min(a[1] + a[3], b[1] + b[3]) - max(a[1], b[1])
    inter = iw * ih if iw > 0 and ih > 0 else 0
    union = a[2] * a[3] + b[2] * b[3] - inter
    return float(inter) > overlap * float(union)


def train_rule(sd, frames, box_frame, boxes, scales, filter_size, cell, K, variant=1, pad=(0, 0), lam=0.01, positive_overlap=0.5,
               negative_overlap=0.3, flip_positives=False, rounds=3, negatives_per_frame=32, mine_overlap=0.5, max_negatives=8192,
               max_iterations=50):
    """sd_hog_train_filter restated with vl_hog_pyramid, hog_box_windows, vl_hog_windows, vl_hog_detect and learn_squared_hinge
    over all frames at once.  -> (filter (D - 1,) float32, bias float32, negatives (n, 4) int32 (frame, level, x, y) in slot
    order, one dict per round with COUNTS and 'solve' (an SvmReport or None); rounds after an early stop are absent)."""
    import torch
    fw, fh = filter_size
    px, py = pad
    S = len(scales)
    f32 = lambda v: float(np.float32(v))                      # the parameters reach the library as floats
    feats, _ = sd.vl_hog_pyramid(frames, scales, cell, K, variant)
    maps, index = [], {}
    for f in range(len(frames)):
        for s in range(S):
            if feats[f][s] is not None:
                index[(f, s)] = len(maps)
                maps.append(feats[f][s])
    size = [(fr.shape[1], fr.shape[0]) for fr in frames]
    pos, unassigned = [], 0
    for f, b in zip(box_frame, boxes):
        lv, _ = sd.hog_box_windows(size[f][0], size[f][1], np.asarray(b)[None], scales, filter_size, cell, K, variant, pad=pad,
                                   positive_overlap=f32(positive_overlap))
        if lv[0, 0] < 0:
            unassigned += 1
            continue
        for fl in range(2 if flip_positives else 1):
            pos.append((index[(int(f), int(lv[0, 0]))], int(lv[0, 1]), int(lv[0, 2]), fl))
    P = sd.vl_hog_windows(maps, np.asarray(pos, np.int32), filter_size, K, variant, pad=pad).cpu().numpy()
    D = P.shape[1]
    # round 0's filter: the float64 mean of the unflipped rows, rounded, minus its float64 mean, rounded
    acc = np.zeros(D - 1)
    n = 0
    for row, w in zip(P, pos):
        if w[3] == 0:
            acc += row[:-1]
            n += 1
    m = (acc / n).astype(np.float32)
    total = 0.0
    for v in m:
        total += float(v)
    filt = (m - np.float32(total / (D - 1))).astype(np.float32)
    bias = np.float32(0.0)
    dd = (D - 1) // (fw * fh)
    frame_boxes = [[tuple(int(v) for v in b) for f, b in zip(box_frame, boxes) if f == i] for i in range(len(frames))]
    cache, reports = [], []
    for rnd in range(rounds + 1):
        rep = dict.fromkeys(COUNTS, 0)
        rep.update(positives=len(pos), unassigned=unassigned)
        free = []
        if cache:
            rows = sd.vl_hog_windows(maps, np.asarray([(index[(f, s)], x, y, 0) for f, s, x, y in cache], np.int32), filter_size, K,
                                     variant, pad=pad).cpu().numpy().astype(np.float64)
            o = rows @ np.concatenate([filt, [bias]]).astype(np.float64)
            free = [k for k in range(len(cache)) if -o[k] >= 1.0]
        thr = -float(np.finfo(np.float32).max) if rnd == 0 else -1.0
        d = sd.vl_hog_detect(frames, scales, torch.from_numpy(filt.reshape(1, dd, fh, fw)), cell, K, thr, variant=variant, bias=[bias],
                             pad=pad, overlap=f32(mine_overlap), max_candidates=8192, max_detections=negatives_per_frame)
        cached = set(cache)
        nf = 0
        for k in range(len(d.frame)):
            f = int(d.frame[k])
            if any(_iou_exceeds(tuple(int(v) for v in d.boxes[k]), b, f32(negative_overlap)) for b in frame_boxes[f]):
                rep["excluded"] += 1
                continue
            rep["mined"] += 1
            v = (f, int(d.level[k]), int(d.cell[k, 0]), int(d.cell[k, 1]))
            if v in cached:
                continue
            if len(cache) < max_negatives:
                cache.append(v)
            elif nf < len(free):
                cached.discard(cache[free[nf]])
                cache[free[nf]] = v
                nf += 1
                rep["evicted"] += 1
            else:
                rep["truncated"] += 1
                continue
            rep["added"] += 1
            cached.add(v)
        rep["cache"] = len(cache)
        rep["solve"] = None
        if rnd > 0 and rep["added"] == 0:
            reports.append(rep)
            break
        win = pos + [(index[(f, s)], x, y, 0) for f, s, x, y in cache]
        A = sd.vl_hog_windows(maps, np.asarray(win, np.int32), filter_size, K, variant, pad=pad)
        y = torch.tensor([1.0] * len(pos) + [-1.0] * len(cache), device=A.device)
        w, srep = sd.learn_squared_hinge(A, y, f32(lam), max_iterations=max_iterations)
        w = w.cpu().numpy()
        filt, bias = w[:-1].copy(), np.float32(w[-1])
        rep["solved"] = 1
        rep["solve"] = srep
        reports.append(rep)
    return filt, bias, np.asarray(cache, np.int32).reshape(-1, 4), reports

"""numpy restatement of the association and the merge of sd_track_detect_faces (include/sd_b200.h):

  - overlap(a, b, t): boxes (x, y, w, h) overlap when float(inter) > t * float(union), inter and union of their pixel
    rectangles in exact integers (inter 0 when they do not meet), compared in float64;
  - associate: a detection of frame f is dropped iff it overlaps the box of an old row of frame f that is alive after the step;
  - merge: within each frame, the alive rows in the order (old rows first, score descending with -0 == +0, row index) are kept
    greedily unless a kept row overlaps them."""
import numpy as np


def overlap(a, b, t: float) -> bool:
    ax, ay, aw, ah = (int(v) for v in a)
    bx, by, bw, bh = (int(v) for v in b)
    iw = min(ax + aw, bx + bw) - max(ax, bx)
    ih = min(ay + ah, by + bh) - max(ay, by)
    inter = iw * ih if iw > 0 and ih > 0 else 0
    union = aw * ah + bw * bh - inter
    return float(inter) > float(t) * float(union)


def associate(det_frame, det_boxes, row_frame, row_boxes, alive, t: float) -> np.ndarray:
    """keep[i]: detection i (of frame det_frame[i]) overlaps no alive row of its frame."""
    rows = {}
    for r, f in enumerate(np.asarray(row_frame)):
        if alive[r]:
            rows.setdefault(int(f), []).append(r)
    return np.array([not any(overlap(row_boxes[r], det_boxes[i], t) for r in rows.get(int(f), []))
                     for i, f in enumerate(np.asarray(det_frame))], dtype=bool)


def merge(frame, boxes, scores, alive, T: int, t: float) -> np.ndarray:
    """The merged alive flags of rows whose first T are old."""
    out = np.array(alive, dtype=bool).copy()
    scores = np.asarray(scores, np.float32)
    for f in np.unique(np.asarray(frame)[out]):
        rows = [r for r in np.flatnonzero(out) if frame[r] == f]
        rows.sort(key=lambda r: (r >= T, -float(scores[r]), r))
        kept = []
        for r in rows:
            if any(overlap(boxes[k], boxes[r], t) for k in kept):
                out[r] = False
            else:
                kept.append(r)
    return out

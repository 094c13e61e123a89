"""Numpy restatements of the tracking rules (include/sd_b200.h, sd_track_boxes and sd_hog_box_scores).

track_box: the face box of a set of landmarks, in float64 with every operation rounded on its own and cvRound as np.rint (ties
to even).  box_crop: the context rectangle of a box, zero outside the frame (np.pad), resized by the oracle's cv::resize
INTER_LINEAR 8-bit rule, which is pinned against cv2."""
import numpy as np

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1


def mean_extent(mean):
    mean = np.asarray(mean, np.float32).ravel()
    L = mean.size // 2
    return (np.float64(mean[:L].min()), np.float64(mean[:L].max()), np.float64(mean[L:].min()), np.float64(mean[L:].max()))


def track_box(x, mean):
    """(x, y, w, h) of the landmarks x (2L floats, [x.., y..]) under the model mean, or None for a degenerate box."""
    x = np.asarray(x, np.float32).ravel()
    L = x.size // 2
    if not np.all(np.isfinite(x)):
        return None
    mx0, mx1, my0, my1 = mean_extent(mean)
    lx0, lx1 = np.float64(x[:L].min()), np.float64(x[:L].max())
    ly0, ly1 = np.float64(x[L:].min()), np.float64(x[L:].max())
    with np.errstate(all="ignore"):
        w = (lx1 - lx0) / (mx1 - mx0)
        h = (ly1 - ly0) / (my1 - my0)
        bx = lx0 - (mx0 + 0.5) * w
        by = ly0 - (my0 + 0.5) * h
    out = []
    for v in (bx, by, w, h):
        r = np.rint(v)
        if not (np.isfinite(r) and INT32_MIN <= r <= INT32_MAX):
            return None
        out.append(int(r))
    return tuple(out) if out[2] >= 1 and out[3] >= 1 else None


def track_boxes(X, mean):
    """(boxes (T, 4) int32, valid (T,) bool) of the rows of X; a degenerate row's box is (0, 0, 0, 0)."""
    X = np.atleast_2d(np.asarray(X, np.float32))
    boxes = np.zeros((X.shape[0], 4), np.int32)
    valid = np.zeros(X.shape[0], bool)
    for t, row in enumerate(X):
        b = track_box(row, mean)
        if b is not None:
            boxes[t], valid[t] = b, True
    return boxes, valid


def context_rect(box, fw, fh):
    """The box with one cell of its scale on every side: (x - ex, y - ey, w + 2 ex, h + 2 ey), e = cvRound of w / fw, h / fh."""
    x, y, w, h = (int(v) for v in box)
    ex, ey = int(np.rint(w / fw)), int(np.rint(h / fh))
    return x - ex, y - ey, w + 2 * ex, h + 2 * ey


def padded_roi(frame, rect):
    """The pixels of rect (x, y, w, h) of a grey frame, 0 outside it (copyMakeBorder BORDER_CONSTANT)."""
    H, W = frame.shape
    x, y, w, h = rect
    pad = max(0, -x, -y, x + w - W, y + h - H)
    p = np.pad(frame, pad)
    return np.ascontiguousarray(p[y + pad:y + pad + h, x + pad:x + pad + w])


def box_crop(oracle, frame, box, fw, fh, cell_size):
    """The (fh + 2) cs x (fw + 2) cs crop sd_hog_box_scores scores for box in frame."""
    roi = padded_roi(frame, context_rect(box, fw, fh))
    return oracle.resize_linear_u8(roi, (fw + 2) * cell_size, (fh + 2) * cell_size)

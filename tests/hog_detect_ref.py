"""A numpy restatement of sd_hog_detections' rule (include/sd_b200.h), in float64 and int64 where the rule says so.

maps: a list of ScoreMap in table order.  For every frame: the candidates (score > threshold, never NaN), ordered by score
descending (floats: -0 == +0) and then by enumeration (map index, q, y, x) with a stable lexsort; the first max_candidates;
their boxes by the exact integer rule; and greedy suppression, (double) inter > overlap * (double) union on int64 areas, where a
box of zero area never suppresses and is never suppressed, up to max_detections kept."""
from collections import namedtuple

import numpy as np

ScoreMap = namedtuple("ScoreMap", "frame level frame_w frame_h level_w level_h scores")   # scores: (Q, height, width) float32

# one detection per row: x, y, w, h, score (float32 bits), filter, level, cell_x, cell_y -- the layout of sd_hog_detection
FIELDS = 9


def rh(n, d):
    """round half up of n / d with floor division, d > 0: floor((2n + d) / (2d)), exact for int64 / Python ints."""
    return (2 * n + d) // (2 * d)


def boxes(x, y, m, cell_size, fw, fh, pad_x, pad_y):
    """(x0, y0, x1, y1) int64 arrays of score positions (x, y) of map m."""
    x = np.asarray(x, np.int64)
    y = np.asarray(y, np.int64)
    sx, sy = np.int64(cell_size) * m.frame_w, np.int64(cell_size) * m.frame_h
    return (rh((x - pad_x) * sx, np.int64(m.level_w)), rh((y - pad_y) * sy, np.int64(m.level_h)),
            rh((x - pad_x + fw) * sx, np.int64(m.level_w)), rh((y - pad_y + fh) * sy, np.int64(m.level_h)))


def suppress(x0, y0, x1, y1, overlap, max_keep):
    """Greedy suppression over boxes in order -> indices kept."""
    area = (x1 - x0) * (y1 - y0)
    kept = []
    for j in range(len(x0)):
        if len(kept) == max_keep:
            break
        if area[j] > 0 and kept:
            k = np.asarray(kept)
            k = k[area[k] > 0]
            iw = np.minimum(x1[k], x1[j]) - np.maximum(x0[k], x0[j])
            ih = np.minimum(y1[k], y1[j]) - np.maximum(y0[k], y0[j])
            inter = np.where((iw > 0) & (ih > 0), iw * ih, 0)
            union = area[k] + area[j] - inter
            if np.any(inter.astype(np.float64) > overlap * union.astype(np.float64)):
                continue
        kept.append(j)
    return np.asarray(kept, np.int64)


def detections(maps, num_frames, cell_size, fw, fh, pad_x, pad_y, threshold, overlap, max_candidates, max_detections):
    """-> (per frame a (k, FIELDS) int32 array of its kept detections in order, above: (num_frames,) int64)."""
    out, above = [], np.zeros(num_frames, np.int64)
    for f in range(num_frames):
        sc, mi, q, y, x = [], [], [], [], []
        for i, m in enumerate(maps):
            if m.frame != f:
                continue
            s = np.asarray(m.scores, np.float32)
            qq, yy, xx = np.nonzero(s > np.float32(threshold))         # C order: q, y, x ascending
            sc.append(s[qq, yy, xx])
            mi.append(np.full(qq.size, i, np.int64))
            q.append(qq)
            y.append(yy)
            x.append(xx)
        if not sc:
            out.append(np.zeros((0, FIELDS), np.int32))
            continue
        sc, mi, q, y, x = (np.concatenate(a) for a in (sc, mi, q, y, x))
        above[f] = sc.size
        order = np.lexsort((np.arange(sc.size), -sc.astype(np.float64)))[:max_candidates]
        sc, mi, q, y, x = sc[order], mi[order], q[order], y[order], x[order]
        b = [np.zeros(sc.size, np.int64) for _ in range(4)]
        for i in np.unique(mi):
            sel = mi == i
            for k, v in enumerate(boxes(x[sel], y[sel], maps[i], cell_size, fw, fh, pad_x, pad_y)):
                b[k][sel] = v
        keep = suppress(*b, overlap, max_detections)
        rec = np.zeros((keep.size, FIELDS), np.int32)
        rec[:, 0] = b[0][keep]
        rec[:, 1] = b[1][keep]
        rec[:, 2] = (b[2] - b[0])[keep]
        rec[:, 3] = (b[3] - b[1])[keep]
        rec[:, 4] = sc[keep].view(np.int32)
        rec[:, 5] = q[keep]
        rec[:, 6] = [maps[i].level for i in mi[keep]]
        rec[:, 7] = x[keep]
        rec[:, 8] = y[keep]
        out.append(rec)
    return out, above

"""A numpy restatement of the part-model rules of include/sd_b200.h, float32 where the rules say fl().

transform: sd_hog_distance_transform of one plane -- the host cost tables in float64 rounded to float32, pass X then pass Y in
float32, each taking candidates in ascending displacement (a non-NaN candidate replaces the best when there is none yet or when
it is strictly greater), so the placement follows the separable tie rule.  part_scores: sd_hog_part_scores' assembly, root
score first and then each part in order.  placements: sd_hog_part_placements' parts of a detection list, boxes by the int64
rule of hog_detect_ref.  brute64: an independent float64 maximum over every (dx, dy), to check the restatement against."""
import numpy as np

from hog_detect_ref import rh

NONE = np.iinfo(np.int64).min


def cost_tables(w, R):
    """(cx, cy) float32 arrays of 2R + 1 entries, index d + R: (float)((double) w0 d d + (double) w1 d), cy with w2, w3."""
    d = np.arange(-R, R + 1, dtype=np.float64)
    w = np.asarray(w, np.float32).astype(np.float64)
    return ((w[0] * d * d + w[1] * d).astype(np.float32), (w[2] * d * d + w[3] * d).astype(np.float32))


def _pass(s, cost, R, axis):
    """One pass along axis (1: X, 0: Y) -> (best float32, chosen displacement int64, NONE where nothing was chosen)."""
    n = s.shape[axis]
    best = np.full(s.shape, -np.inf, np.float32)
    arg = np.full(s.shape, NONE, np.int64)
    idx = np.arange(n)
    with np.errstate(invalid="ignore"):
        for d in range(-R, R + 1):
            src = idx + d
            ok = (src >= 0) & (src < n)
            cand = np.full(s.shape, np.nan, np.float32)
            if axis == 1:
                cand[:, ok] = s[:, src[ok]] - cost[d + R]
            else:
                cand[ok, :] = s[src[ok], :] - cost[d + R]
            take = ~np.isnan(cand) & ((arg == NONE) | (cand > best))
            best = np.where(take, cand, best)
            arg = np.where(take, d, arg)
    return best, arg


def transform(s, w, R):
    """-> (D (h, w) float32, placements (h, w, 2) int32 of (u, v), (-1, -1) for none)."""
    s = np.asarray(s, np.float32)
    h, W = s.shape
    cx, cy = cost_tables(w, R)
    t, dx = _pass(s, cx, R, 1)
    D, ey = _pass(t, cy, R, 0)
    place = np.full((h, W, 2), -1, np.int32)
    v, u = np.nonzero(ey != NONE)
    row = v + ey[v, u]
    ok = dx[row, u] != NONE
    place[v[ok], u[ok], 0] = u[ok] + dx[row[ok], u[ok]]
    place[v[ok], u[ok], 1] = row[ok]
    return D, place


def brute64(s, w, R):
    """float64 maximum of s(v + dy, u + dx) - cx64[dx] - cy64[dy] over the window (NaN skipped; -inf where all are NaN) and,
    per position, the float64 gap between the best and the second best candidate (inf when there is one)."""
    s = np.asarray(s, np.float64)
    h, W = s.shape
    cx, cy = (c.astype(np.float64) for c in cost_tables(w, R))
    best = np.full((h, W), -np.inf)
    second = np.full((h, W), -np.inf)
    where = np.full((h, W, 2), -1, np.int64)
    for dy in range(-R, R + 1):
        for dx in range(-R, R + 1):
            if abs(dy) >= h or abs(dx) >= W:
                continue
            c = np.full((h, W), np.nan)
            ys, xs = slice(max(0, -dy), min(h, h - dy)), slice(max(0, -dx), min(W, W - dx))
            ysrc, xsrc = slice(max(0, dy), min(h, h + dy)), slice(max(0, dx), min(W, W + dx))
            c[ys, xs] = s[ysrc, xsrc] - cx[dx + R] - cy[dy + R]
            c = np.where(np.isnan(c), -np.inf, c)
            up = c > best
            second = np.where(up, best, np.maximum(second, c))
            uu, vv = np.meshgrid(np.arange(W), np.arange(h))
            where[..., 0] = np.where(up, uu + dx, where[..., 0])
            where[..., 1] = np.where(up, vv + dy, where[..., 1])
            best = np.where(up, c, best)
    return best, best - second, where


def part_scores(root, D, anchors, pad, part_pad):
    """root (Q, oh, ow) float32, D (Q * P, ph, pw) float32 (or None: no part map), anchors (Q, P, 2) -> (Q, oh, ow) float32."""
    root = np.asarray(root, np.float32)
    Q, oh, ow = root.shape
    P = anchors.shape[1]
    ph, pw = (0, 0) if D is None else D.shape[1:]
    y, x = np.meshgrid(np.arange(oh), np.arange(ow), indexing="ij")
    out = np.empty_like(root)
    for q in range(Q):
        total = root[q].copy()
        outside = np.zeros((oh, ow), bool)
        for p in range(P):
            u0 = 2 * (x - pad[0]) + int(anchors[q, p, 0]) + part_pad[0]
            v0 = 2 * (y - pad[1]) + int(anchors[q, p, 1]) + part_pad[1]
            ok = (u0 >= 0) & (u0 < pw) & (v0 >= 0) & (v0 < ph)
            outside |= ~ok
            if ok.any():
                total[ok] = total[ok] + D[q * P + p][v0[ok], u0[ok]]
        out[q] = np.where(outside, np.float32(-np.inf), total)
    return out


def placements(rec, pmap, anchors, pad, part_pad, part_size, cell_size):
    """Parts of one detection record (hog_detect_ref layout) -> (P, 7) int32 rows (u, v, term bits, x, y, w, h).

    pmap: dict with 'D' (Q * P, ph, pw) and 'place' (Q * P, ph, pw, 2) of the transform (or None for no part map), frame_w,
    frame_h, part_level_w, part_level_h."""
    q, cx, cy = int(rec[5]), int(rec[7]), int(rec[8])
    P = anchors.shape[1]
    out = np.zeros((P, 7), np.int32)
    for p in range(P):
        u0 = 2 * (cx - pad[0]) + int(anchors[q, p, 0]) + part_pad[0]
        v0 = 2 * (cy - pad[1]) + int(anchors[q, p, 1]) + part_pad[1]
        row = [-1, -1, np.float32(-np.inf).view(np.int32), 0, 0, 0, 0]
        D = pmap["D"]
        if D is not None and 0 <= u0 < D.shape[2] and 0 <= v0 < D.shape[1]:
            u, v = (int(t) for t in pmap["place"][q * P + p, v0, u0])
            row[2] = np.float32(D[q * P + p, v0, u0]).view(np.int32)
            if u >= 0:
                sx, sy = cell_size * pmap["frame_w"], cell_size * pmap["frame_h"]
                x0, x1 = rh((u - part_pad[0]) * sx, pmap["part_level_w"]), rh((u - part_pad[0] + part_size[0]) * sx, pmap["part_level_w"])
                y0, y1 = rh((v - part_pad[1]) * sy, pmap["part_level_h"]), rh((v - part_pad[1] + part_size[1]) * sy, pmap["part_level_h"])
                row[0:2] = [u, v]
                row[3:7] = [x0, y0, x1 - x0, y1 - y0]
        out[p] = row
    return out

"""The sample-warp rule of sd_hog_batch_warped (include/sd_b200.h, sd_sample_warp) restated in numpy: a P x P window of the
virtual frame V = cv2.warpAffine(g, M, (Wv, Hv), INTER_LINEAR | WARP_INVERSE_MAP, BORDER_CONSTANT, 0), computed pixel by pixel
from g by face_chip_ref's fixed-point arithmetic at V's own coordinates, with 0 outside [0, Wv) x [0, Hv) (copyMakeBorder on V)."""
import numpy as np

import face_chip_ref as R


def materialise(g, M, size):
    """V itself, by cv2 (the reference every test compares against)."""
    import cv2
    return cv2.warpAffine(g, np.asarray(M, np.float64), (int(size[0]), int(size[1])), flags=cv2.INTER_LINEAR | cv2.WARP_INVERSE_MAP,
                          borderMode=cv2.BORDER_CONSTANT, borderValue=0)


def window(g, M, size, x0, y0, P):
    """The (P, P) uint8 window [x0, x0 + P) x [y0, y0 + P) of V (g: (H, W) uint8), or None when the warp is invalid."""
    g = np.asarray(g, np.uint8)
    M = np.asarray(M, np.float64)
    Wv, Hv = int(size[0]), int(size[1])
    if Wv < 1 or Hv < 1 or not np.all(np.isfinite(M)) or R.taps(M, Wv, Hv, g.shape[1], g.shape[0]) is None:
        return None
    out = np.zeros((P, P), np.uint8)
    u0, u1, v0, v1 = max(x0, 0), min(x0 + P, Wv), max(y0, 0), min(y0 + P, Hv)
    if u0 >= u1 or v0 >= v1:
        return out
    X, Y = np.arange(u0, u1, dtype=np.float64), np.arange(v0, v1, dtype=np.float64)
    ad, bd = np.rint(M[0, 0] * X * 1024).astype(np.int64), np.rint(M[1, 0] * X * 1024).astype(np.int64)
    X0 = np.rint((M[0, 1] * Y + M[0, 2]) * 1024).astype(np.int64) + 16
    Y0 = np.rint((M[1, 1] * Y + M[1, 2]) * 1024).astype(np.int64) + 16
    sx, sy = (X0[:, None] + ad[None, :]) >> 5, (Y0[:, None] + bd[None, :]) >> 5
    xs, ys, fx, fy = sx >> 5, sy >> 5, sx & 31, sy & 31
    H, W = g.shape

    def tap(dy, dx):
        yy, xx = ys + dy, xs + dx
        inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        return np.where(inside, g[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)], 0).astype(np.int64)

    acc = tap(0, 0) * ((32 - fx) * (32 - fy) * 32) + tap(0, 1) * (fx * (32 - fy) * 32) + tap(1, 0) * ((32 - fx) * fy * 32) + \
        tap(1, 1) * (fx * fy * 32)
    out[v0 - y0:v1 - y0, u0 - x0:u1 - x0] = np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)
    return out


def crop(V, x0, y0, P):
    """The (P, P) window of a materialised V with zero padding (copyMakeBorder BORDER_CONSTANT 0)."""
    Hv, Wv = V.shape
    out = np.zeros((P, P), np.uint8)
    u0, u1, v0, v1 = max(x0, 0), min(x0 + P, Wv), max(y0, 0), min(y0 + P, Hv)
    if u0 < u1 and v0 < v1:
        out[v0 - y0:v1 - y0, u0 - x0:u1 - x0] = V[v0:v1, u0:u1]
    return out

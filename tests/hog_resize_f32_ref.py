"""The float pyramid's resize rule (sd_hog_pyramid_float, include/sd_b200.h), restated in numpy.

cv::resize INTER_LINEAR of float frames, channel by channel, in float32 with every product and every sum rounded on its own (numpy
never fuses them).  tests/test_hog_pyramid_float_oracle.py checks it against cv2.resize; the GPU tests check the library against it."""
import numpy as np


def taps(n_out: int, n_in: int):
    """(s, f) per output coordinate of an n_in -> n_out px axis: scale = 1 / (n_out / n_in) in double, f = (float)((d + 0.5) *
    scale - 0.5), s = floor(f), f -= s in float32."""
    scale = 1.0 / (n_out / n_in)
    f = ((np.arange(n_out, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    return s, (f - s.astype(np.float32)).astype(np.float32)


def resize_f32(frame, lw: int, lh: int, skip_zero_taps: bool = False):
    """The lh x lw level of a float32 (H, W) or (H, W, C) frame.  skip_zero_taps: a deliberately wrong variant that leaves out
    the column taps of weight 0, for the tests that must tell it apart."""
    src = np.asarray(frame, dtype=np.float32)
    H, W = src.shape[:2]
    if lw == W and lh == H:
        return src.copy()                            # a bit copy: NaN payloads and -0 kept
    S = src.reshape(H, W, -1)
    sx, fx = taps(lw, W)
    fx = np.where(sx < 0, np.float32(0), fx)
    sx = np.maximum(sx, 0)
    last = sx >= W - 1
    fx = np.where(last, np.float32(0), fx).astype(np.float32)
    sx = np.where(last, W - 1, sx)
    a0, a1 = (np.float32(1) - fx)[:, None], fx[:, None]
    with np.errstate(invalid="ignore", over="ignore"):
        t = S[:, sx, :] * a0                         # (H, lw, C)
        right = S[:, np.minimum(sx + 1, W - 1), :] * a1
        two = ~last if not skip_zero_taps else (~last & (fx != 0))
        t = np.where(two[None, :, None], t + right, t).astype(np.float32)
        sy, fy = taps(lh, H)
        y0, y1 = np.clip(sy, 0, H - 1), np.clip(sy + 1, 0, H - 1)
        b0, b1 = (np.float32(1) - fy)[:, None, None], fy[:, None, None]
        out = (t[y0] * b0 + t[y1] * b1).astype(np.float32)
    return out.reshape((lh, lw) + src.shape[2:])


def level_size(w: int, h: int, s: float):
    """(level_w, level_h) of a w x h frame at scale s: floor(w s + 0.5), floor(h s + 0.5) in double."""
    return int(np.floor(w * s + 0.5)), int(np.floor(h * s + 0.5))

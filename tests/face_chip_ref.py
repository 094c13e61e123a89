"""The face chip rule of sd_face_chips (include/sd_b200.h) restated in numpy.

fit: the least-squares similarity T(u) = [[a, -b], [b, a]] u + t from template points u (chip pixels) to a face's landmarks,
float64 with sums in list order and every operation rounded on its own.  warp: cv2.warpAffine(frame, M, (w, h), INTER_LINEAR |
WARP_INVERSE_MAP, BORDER_CONSTANT, 0) with M the chip-to-frame matrix: 10-bit fixed-point coordinates, a 1/32 px tap grid, 15-bit
integer weights for 8-bit frames and float weights summed left to right for float frames.  Chips are (h, w, C), channels last."""
import numpy as np

INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
INT16_MIN, INT16_MAX = -2 ** 15, 2 ** 15 - 1


def template(mean, width, height, padding=0.25, landmarks=None):
    """The default template of sd_face_chip_template: ((m + 0.5 + padding) / (1 + 2 padding)) * side per axis, (n, 2) float64."""
    mean = np.asarray(mean, np.float32).ravel()
    L = mean.size // 2
    idx = np.arange(L) if landmarks is None else np.asarray(landmarks, np.int64)
    den = 1.0 + 2.0 * padding
    tx = (mean[idx].astype(np.float64) + 0.5 + padding) / den * width
    ty = (mean[L + idx].astype(np.float64) + 0.5 + padding) / den * height
    return np.stack([tx, ty], axis=1)


def fit(x, landmark_index, tmpl):
    """(a, b, tx, ty) of the similarity from tmpl ((n, 2) float64) to the landmarks landmark_index of x (2L float32, [x.., y..]),
    or None when a used landmark is not finite, den == 0 or a^2 + b^2 == 0."""
    x = np.asarray(x, np.float32).ravel()
    L = x.size // 2
    idx = np.asarray(landmark_index, np.int64)
    px, py = x[idx].astype(np.float64), x[L + idx].astype(np.float64)
    if not (np.all(np.isfinite(px)) and np.all(np.isfinite(py))):
        return None
    u = np.asarray(tmpl, np.float64)
    n = len(idx)
    with np.errstate(all="ignore"):
        sux = suy = sxx = sxy = 0.0
        for k in range(n):
            sux += u[k, 0]; suy += u[k, 1]; sxx += px[k]; sxy += py[k]
        ux, uy, mx, my = sux / n, suy / n, sxx / n, sxy / n
        den = num_a = num_b = 0.0
        for k in range(n):
            dux, duy, dx, dy = u[k, 0] - ux, u[k, 1] - uy, px[k] - mx, py[k] - my
            den += dux * dux + duy * duy
            num_a += dux * dx + duy * dy
            num_b += dux * dy - duy * dx
        if den == 0:
            return None
        a, b = num_a / den, num_b / den
        if a * a + b * b == 0:
            return None
        tx = mx - (a * ux - b * uy)
        ty = my - (b * ux + a * uy)
    return a, b, tx, ty


def matrices(a, b, tx, ty):
    """(chip_to_frame, frame_to_chip), two 2 x 3 float64 matrices: [a, -b, tx; b, a, ty] and its exact algebraic inverse."""
    s = a * a + b * b
    ia, ib = a / s, b / s
    itx = -(ia * tx + ib * ty)
    ity = ib * tx - ia * ty
    return np.array([[a, -b, tx], [b, a, ty]]), np.array([[ia, ib, itx], [-ib, ia, ity]])


def _round(v):
    """cvRound of float64 values (ties to even) as int64, or None when one is not finite or leaves int32."""
    with np.errstate(all="ignore"):
        r = np.rint(v)
    if not np.all(np.isfinite(r)) or r.min() < INT32_MIN or r.max() > INT32_MAX:
        return None
    return r.astype(np.int64)


def taps(M, width, height, frame_w, frame_h):
    """((ys, xs), (fy, fx)) of every chip pixel: the top-left tap and its 1/32 fractions, each (h, w) int64; None when a
    fixed-point coordinate leaves int32, or a tap coordinate leaves int16 in a frame wider or taller than 32,767 px."""
    X, Y = np.arange(width, dtype=np.float64), np.arange(height, dtype=np.float64)
    adelta, bdelta = _round(M[0, 0] * X * 1024), _round(M[1, 0] * X * 1024)
    x0, y0 = _round((M[0, 1] * Y + M[0, 2]) * 1024), _round((M[1, 1] * Y + M[1, 2]) * 1024)
    if adelta is None or bdelta is None or x0 is None or y0 is None:
        return None
    x0, y0 = x0 + 16, y0 + 16
    sx, sy = x0[:, None] + adelta[None, :], y0[:, None] + bdelta[None, :]
    for v in (x0, y0, sx, sy):
        if v.min() < INT32_MIN or v.max() > INT32_MAX:
            return None
    sx, sy = sx >> 5, sy >> 5
    xs, ys = sx >> 5, sy >> 5
    if max(frame_w, frame_h) > INT16_MAX and (min(xs.min(), ys.min()) < INT16_MIN or max(xs.max(), ys.max()) > INT16_MAX):
        return None
    return (ys, xs), (sy & 31, sx & 31)


def warp(frame, M, width, height):
    """The (height, width, C) chip of frame ((H, W) or (H, W, C), uint8 or float32) under the chip-to-frame matrix M, or None
    when taps() refuses M."""
    f = np.asarray(frame)
    f3 = f[:, :, None] if f.ndim == 2 else f
    H, W, C = f3.shape
    t = taps(M, width, height, W, H)
    if t is None:
        return None
    (ys, xs), (fy, fx) = t

    def tap(dy, dx):
        yy, xx = ys + dy, xs + dx
        inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = f3[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        return np.where(inside[..., None], v, np.zeros((), f3.dtype))

    s00, s01, s10, s11 = tap(0, 0), tap(0, 1), tap(1, 0), tap(1, 1)
    fx, fy = fx[..., None], fy[..., None]
    if f3.dtype == np.uint8:
        w0, w1, w2, w3 = (32 - fx) * (32 - fy) * 32, fx * (32 - fy) * 32, (32 - fx) * fy * 32, fx * fy * 32
        acc = s00.astype(np.int64) * w0 + s01 * w1 + s10 * w2 + s11 * w3
        return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)
    wx0, wx1 = (1 - fx / 32).astype(np.float32), (fx / 32).astype(np.float32)
    wy0, wy1 = (1 - fy / 32).astype(np.float32), (fy / 32).astype(np.float32)
    with np.errstate(all="ignore"):
        return s00 * (wx0 * wy0) + s01 * (wx1 * wy0) + s10 * (wx0 * wy1) + s11 * (wx1 * wy1)


def face_chips(frames, face_frame, landmarks, landmark_index, tmpl, width, height):
    """sd_face_chips of a list of frames: (chips (n, h, w, C), chip_to_frame (n, 2, 3), frame_to_chip (n, 2, 3), valid (n,)
    bool).  An invalid face has a zero chip and zero transforms."""
    n = len(face_frame)
    f0 = np.asarray(frames[0])
    C = 1 if f0.ndim == 2 else f0.shape[2]
    chips = np.zeros((n, height, width, C), f0.dtype)
    c2f, f2c = np.zeros((n, 2, 3)), np.zeros((n, 2, 3))
    valid = np.zeros(n, bool)
    for i in range(n):
        p = fit(landmarks[i], landmark_index, tmpl)
        if p is None:
            continue
        M, Mi = matrices(*p)
        chip = warp(frames[face_frame[i]], M, width, height)
        if chip is None:
            continue
        chips[i], c2f[i], f2c[i], valid[i] = chip, M, Mi, True
    return chips, c2f, f2c, valid

"""Float64 truth, per-element error bars and a float32 kernel-order restatement for VLFeat's HOG (hog.c's vl_hog_put_image,
vl_hog_put_polar_field and vl_hog_extract) as the landmark kernels (csrc/sd_hog.cu) and the dense kernels (csrc/sd_hog_dense.cu)
compute it.

Discrete decisions are inputs.  A pixel's orientation bin or bins, and for multi-channel frames the channel whose gradient wins,
are decided by the float32 chain that hog.c and the kernels share operation for operation (`image_pixels`, `polar_pixels`).
For 8-bit grey frames those bins equal oracle.hog_orientation_bins, which the exhaustive orientation tests pin to the kernels'
bins for every (gx, gy).  For float frames and polar fields the builders also assert that every decision has a float64 margin
far beyond float32 rounding (MARGIN times the decision's own error bound), so that float64 would make the same decisions.  The
truth then computes every value in float64 from the float32 inputs:

    m        gradient modulus sqrt(gx^2 + gy^2) of the winning channel (the polar modulus as given)
    w_o      orientation weight: 1 (nearest bin); bilinear w1 = acos(s0) / (pi / K), w0 = 1 - w1 with s0 the top |<u, o_k>|;
             polar bilinear w1 = frac(angle / (pi / K))
    wx, wy   spatial weights of hog.c:697-709, h = (t + 0.5) / cs - 0.5, w2 = h - floor(h), w1 = 1 - w2
    vote     m * wx * wy * w_o^2 into cells (bx, by) .. (bx + 1, by + 1) inside the grid
    hist     the sum of a cell's votes per bin; energy E = sum_k (h_k + h_{k+K})^2; block factors 1 / sqrt(sum of 4 E + 1e-4)
             over blocks clamped to the grid; min(0.2, f h) per factor; UoCTTI (0.5 * sums, texture dims sum_k hc_q / sqrt 18)
             or Dalal-Triggs projections, in VLFeat's planar layout [dd][hogH][hogW].

Bars.  Each float64 quantity carries an absolute bound on the float32 computation's error (u = 2^-24, first order):
  - modulus: 8-bit gradients are exact integers, so one rounding of the root (u m).  Float frames: each difference of two float32
    operands is one correctly rounded subtraction (u |g|), then the squares, the sum and the root: 3u m;
  - spatial weights: hog_spatial_weight is a deterministic function of the coordinate (one rounding of h, an exact h - b, one
    rounding of 1 - w2), so each bar is that rounding evaluated at the coordinate, |w32 - w| (at most u |h| + u, 0 where exact);
  - bilinear orientation weights: the float32 top score s0 is an input, restated operation for operation as hog_bins_bilinear
    computes it, and w1 = acos(s0) / (pi / K) in float64 from it; the float roundings of acos and of the quotient (and hog.c's
    acosf) give 3u w1, and w0 = 1 - w1 one more u w0.  Polar: ho is one rounding, u |ho|, and wo1 = 1 - wo2 one more u;
  - vote: the factors' bars carried through the product, plus 4u for the products' roundings;
  - histogram bin: the votes' bars summed, plus a random walk over the n votes' additions, LAMBDA sqrt(n) u hist, with the
    probabilistic factor LAMBDA = 8 applied once (as in gemm_ref.py and chol_ref.py);
  - energy: 2 |h_k + h_{k+K}| (e_k + e_{k+K}) per k, plus (2K + 2) u E for its float roundings; block factor f = s^-1/2 moves by
    f e_s / (2 s); haf = f ha by f e_ha + ha e_f; the clamp at 0.2 is 1-Lipschitz (and exact when the truth is clamped by more
    than its bar); sums add their bars; the final store adds 2u |value| (u for the rounding, u of room for the double chain);
    the texture constant (float 1 / sqrtf(18)) 3u.
  Measured on the frames of the tests, the bar of a feature is a median 50 to 180 u of its value (99th percentile up to about
  1100 u, in polar bilinear cells whose ho is large).
A feature whose truth and bar are both 0 (a cell without votes) must be exactly 0.

`emulate` restates the kernels' float32 vote order: per cell column and row, T[b] = sum over the row's pixels, x ascending, of
g * wx (bilinear: (g * (wx * w_o)) * w_o per bin, the first bin first), then per cell hist[b] = sum over rows, y ascending, of
T[b] * wy; the energy in float, block factors and projections in double as hog_cell_factors / hog_cell_features.  It is what
the bars are tested against on the CPU, and its `defect` argument plants the defects they must reject.
"""
import math

import numpy as np

U = 2.0 ** -24
LAMBDA = 8.0
MARGIN = 16.0                 # a decision's float64 margin must exceed MARGIN times its float32 error bound
f32 = np.float32


def grid(W, H, cs):
    """(hogW, hogH) of hog.c:542-543."""
    return (W + cs // 2) // cs, (H + cs // 2) // cs


def dims(variant, K):
    return 3 * K + 4 if variant == 1 else 4 * K


def orientations(K):
    """hog.c:195-204: (cos, sin)(k pi / K) computed in double and rounded to float."""
    a = np.arange(K) * math.pi / K
    return np.cos(a).astype(f32), np.sin(a).astype(f32)


# ---- per-pixel decisions and values --------------------------------------------------------------------------------------
class Pixels:
    """The votes of an H x W frame: moduli m (float64 truth, its bar em, the kernel's float32 value m32) and one or two
    orientation entries (bins, weight truth, bar, float32 weight).  bins -1: no vote."""

    def __init__(self, m, em, m32, bins, wo=None, ewo=None, wo32=None):
        self.m, self.em, self.m32 = m, em, m32
        self.bins = list(bins)
        one = np.ones(m.shape)
        self.wo = list(wo) if wo is not None else [one]
        self.ewo = list(ewo) if ewo is not None else [np.zeros(m.shape)]
        self.wo32 = list(wo32) if wo32 is not None else [one.astype(f32)]
        self.bilinear = len(self.bins) == 2

    @property
    def shape(self):
        return self.m.shape


def _scores32(ux, uy, K):
    """|<u, o_k>| and the directed bins of every k, in the reference's float32 chain (hog.c:656-672)."""
    ox, oy = orientations(K)
    s = (ux[None] * ox[:, None, None]).astype(f32) + (uy[None] * oy[:, None, None]).astype(f32)
    s = s.astype(f32)
    b = np.arange(K)[:, None, None] + np.where(s < 0, K, 0)
    return np.abs(s), b


def _top_two(s, b):
    """hog.c's top-two tracking: a score replaces the first only when strictly larger, else the second when strictly larger;
    returns (s0, b0, s1, b1) with -1 bins where no score is positive."""
    K = s.shape[0]
    s0 = np.zeros(s.shape[1:], f32); s1 = np.zeros_like(s0)
    b0 = np.full(s.shape[1:], -1); b1 = np.full(s.shape[1:], -1)
    for k in range(K):
        first = s[k] > s0
        second = ~first & (s[k] > s1)
        b1 = np.where(first, b0, np.where(second, b[k], b1))
        s1 = np.where(first, s0, np.where(second, s[k], s1))
        b0 = np.where(first, b[k], b0)
        s0 = np.where(first, s[k], s0)
    return s0, b0, s1, b1


def decision_doubt(frame, K, bilinear):
    """Mask of the voting pixels of a frame (C, H, W) whose channel or orientation decision is in doubt: the float64 lead of the
    winning channel's g2, of the top |<u, o_k>| over the next (bilinear: also of the second over the third) and the second's
    distance from 0 (its sign) must each exceed MARGIN times the float32 error bound of the quantities compared."""
    x = np.asarray(frame).astype(np.float64)
    if x.ndim == 2:
        x = x[None]
    C, H, W = x.shape
    gx = np.zeros(x.shape); gy = np.zeros(x.shape); dg = np.zeros(x.shape)
    gx[:, 1:-1, 1:-1] = x[:, 1:-1, 2:] - x[:, 1:-1, :-2]
    gy[:, 1:-1, 1:-1] = x[:, 2:, 1:-1] - x[:, :-2, 1:-1]
    dg[:, 1:-1, 1:-1] = U * (np.abs(x[:, 1:-1, 2:]) + np.abs(x[:, 1:-1, :-2]) + np.abs(x[:, 2:, 1:-1]) + np.abs(x[:, :-2, 1:-1]))
    g2 = gx ** 2 + gy ** 2
    vote = np.max(g2, axis=0) > 0
    bad = np.zeros((H, W), bool)
    cc = np.argmax(g2, axis=0)
    if C > 1:
        srt = np.sort(g2, axis=0)
        eg2 = np.max(2 * np.sqrt(g2) * dg + 4 * U * g2, axis=0)
        bad |= srt[-1] - srt[-2] <= MARGIN * 2 * eg2
    yy, xx = np.mgrid[0:H, 0:W]
    m = np.where(vote, np.sqrt(g2[cc, yy, xx]), 1.0)
    ds = 6 * U + 2 * dg[cc, yy, xx] / m
    a = np.arange(K) * math.pi / K
    s = np.abs((gx[cc, yy, xx] / m)[None] * np.cos(a)[:, None, None] + (gy[cc, yy, xx] / m)[None] * np.sin(a)[:, None, None])
    s = np.sort(s, axis=0)[::-1]
    need = MARGIN * (ds + 2 * U)
    if K > 1:
        bad |= s[0] - s[1] <= need
        if bilinear:
            bad |= s[1] - (s[2] if K > 2 else 0.0) <= need
    return bad & vote


def image_pixels(frame, K, bilinear=False, check_margin=None):
    """Votes of a frame (H, W) or planar (C, H, W), uint8 or float32, as vl_hog_put_image (hog.c:616-682).  Interior pixels
    vote; the channel with the largest float32 g2 wins (strictly, from 0).  check_margin (default: float frames) asserts that
    every decision has a float64 margin of MARGIN times its bar."""
    img = np.asarray(frame)
    if img.ndim == 2:
        img = img[None]
    is_u8 = img.dtype == np.uint8
    if check_margin is None:
        check_margin = not is_u8
    x = img.astype(f32)
    C, H, W = x.shape
    inner = (slice(None), slice(1, H - 1), slice(1, W - 1))
    gx32 = np.zeros(x.shape, f32); gy32 = np.zeros(x.shape, f32)
    gx32[inner] = x[:, 1:-1, 2:] - x[:, 1:-1, :-2]
    gy32[inner] = x[:, 2:, 1:-1] - x[:, :-2, 1:-1]
    g2c = ((gx32 * gx32).astype(f32) + (gy32 * gy32).astype(f32)).astype(f32)
    # winning channel: first strict maximum of g2 from 0
    ch = np.full((H, W), -1)
    best = np.zeros((H, W), f32)
    for c in range(C):
        take = g2c[c] > best
        ch = np.where(take, c, ch)
        best = np.where(take, g2c[c], best)
    vote = ch >= 0
    cc = np.maximum(ch, 0)
    yy, xx = np.mgrid[0:H, 0:W]
    gx = gx32[cc, yy, xx]; gy = gy32[cc, yy, xx]
    m32 = np.sqrt(best).astype(f32)
    # float64 values and bars
    x64 = x.astype(np.float64)
    gx64 = np.zeros(x.shape); gy64 = np.zeros(x.shape)
    gx64[inner] = x64[:, 1:-1, 2:] - x64[:, 1:-1, :-2]
    gy64[inner] = x64[:, 2:, 1:-1] - x64[:, :-2, 1:-1]
    g2_64 = gx64 ** 2 + gy64 ** 2
    m = np.where(vote, np.sqrt(g2_64[cc, yy, xx]), 0.0)
    # 8-bit: the gradient and its square are exact integers, one rounding of the root.  Float: each difference of two float32
    # operands is one correctly rounded subtraction (u |g|), then the squares, the sum and the root.
    em = np.where(vote, (U if is_u8 else 3 * U) * m, 0.0)
    # unit vector (g >= 1e-10 here: hog_unit is a float division) and scores in float32
    mm = np.where(vote, m32, f32(1))
    assert np.all(~vote | (m32.astype(np.float64) > 1e-10)), "moduli below the 1e-10 floor are out of scope"
    ux = (gx / mm).astype(f32); uy = (gy / mm).astype(f32)
    s, b = _scores32(ux, uy, K)
    s0, b0, s1, b1 = _top_two(s, b)
    b0 = np.where(vote, b0, -1); b1 = np.where(vote, b1, -1)
    if check_margin:
        bad = decision_doubt(img, K, bilinear)
        assert not bad.any(), f"{int(bad.sum())} decisions lie within the float32 margin"
    if not bilinear:
        return Pixels(m, em, np.where(vote, m32, f32(0)), [b0])
    # The float32 top score s0 is an input, like the bins (the float32 restatement of hog_bins_bilinear above): w1 =
    # acos(s0) / (pi / K) in float64 from it.  The kernels round acos to float and the quotient to float, hog.c takes acosf:
    # 3u w1.  w0 = 1 - w1 is one more float subtraction (u w0).
    pi_k = math.pi / K
    s0c = np.minimum(s0, f32(1)).astype(np.float64)
    w1_32 = (np.arccos(s0c).astype(f32).astype(np.float64) / pi_k).astype(f32)
    w1 = np.where(vote, np.arccos(s0c) / pi_k, 0.0)
    ew1 = np.where(vote, 3 * U * w1, 0.0)
    ew0 = np.where(vote, ew1 + U * (1.0 - w1), 0.0)
    return Pixels(m, em, np.where(vote, m32, f32(0)), [b0, b1], [1.0 - w1, w1], [ew0, ew1],
                  [(f32(1) - w1_32).astype(f32), w1_32])


def polar_pixels(modulus, angle, K, directed=True, bilinear=False):
    """Votes of a polar field (vl_hog_put_polar_field, hog.c:770-800, as polar_bins restates it): every pixel with a modulus
    > 0 votes; ho = angle / (pi / K).  Asserts each decision's float64 margin."""
    mod = np.asarray(modulus, f32); ang = np.asarray(angle, f32)
    pi_k = math.pi / K
    period = 2 * K if directed else K
    ho32 = (ang.astype(np.float64) / pi_k).astype(f32)
    bino32 = np.floor(ho32)
    wo2_32 = (ho32 - bino32).astype(f32)
    wo1_32 = (f32(1) - wo2_32).astype(f32)
    r = np.mod(bino32, period).astype(np.int64)
    ho = ang.astype(np.float64) / pi_k
    frac = ho - np.floor(ho)
    eho = U * (np.abs(ho) + 1)                                  # the decisions' error bound
    vote = mod > 0
    ok = (np.floor(ho) == bino32) & (frac > MARGIN * eho) & (frac < 1 - MARGIN * eho)
    if not bilinear:
        ok &= np.abs(frac - 0.5) > MARGIN * eho
    assert np.all(~vote | ok), f"{int(np.sum(vote & ~ok))} polar decisions lie within the float32 margin"
    m = np.where(vote, mod.astype(np.float64), 0.0)
    m32 = np.where(vote, mod, f32(0))
    em = np.zeros(mod.shape)
    if not bilinear:
        b = np.where(wo1_32 > wo2_32, r, (r + 1) % period)
        return Pixels(m, em, m32, [np.where(vote, b, -1)])
    # bilinear weights: ho is one rounding (u |ho|), wo2 = ho - bino is then exact, wo1 = 1 - wo2 one more rounding (u)
    b1 = (r + 1) % period
    ew1 = np.where(vote, U * np.abs(ho), 0.0)
    ew0 = np.where(vote, U * (np.abs(ho) + 1), 0.0)
    return Pixels(m, em, m32, [np.where(vote, r, -1), np.where(vote, b1, -1)], [1.0 - frac, frac], [ew0, ew1], [wo1_32, wo2_32])


# ---- spatial weights -------------------------------------------------------------------------------------------------------
def spatial64(n, cs):
    """Per coordinate t < n: cell b, weights w1, w2 in float64 and their bars (hog.c:697-709).  The float32 weights are
    deterministic functions of t and cs (one rounding of h, an exact h - b, one rounding of 1 - w2), so each bar is that
    rounding evaluated at the coordinate: |w32 - w| (at most u |h| for w2 and u |h| + u for w1; 0 where h is exact)."""
    h = (np.arange(n) + 0.5) / cs - 0.5
    b = np.floor(h)
    b32, w1_32, w2_32 = spatial32(n, cs)
    assert np.array_equal(b32, b), "a spatial cell decision differs in float32"
    w2 = h - b
    w1 = 1.0 - w2
    return b.astype(np.int64), w1, w2, np.abs(w1_32 - w1), np.abs(w2_32 - w2)


def spatial32(n, cs):
    """hog_spatial_weight: h rounded from double, w2 = h - b in float, w1 = (float)(1 - (double)w2)."""
    h = ((np.arange(n) + 0.5) / cs - 0.5).astype(f32)
    b = np.floor(h)
    w2 = (h - b).astype(f32)
    w1 = (1.0 - w2.astype(np.float64)).astype(f32)
    return b.astype(np.int64), w1, w2


# ---- histograms ------------------------------------------------------------------------------------------------------------
def hist64(px, cs, K):
    """Float64 histograms [2K][hogH][hogW], their bars, and per-bin vote counts."""
    H, W = px.shape
    cw, ch = grid(W, H, cs)
    bx, wx1, wx2, ewx1, ewx2 = spatial64(W, cs)
    by, wy1, wy2, ewy1, ewy2 = spatial64(H, cs)
    nbin = 2 * K * ch * cw
    hist = np.zeros(nbin); err = np.zeros(nbin); cnt = np.zeros(nbin)
    for b, wo, ewo in zip(px.bins, px.wo, px.ewo):
        sel = b >= 0
        yy, xx = np.nonzero(sel)
        bb, m, em = b[sel], px.m[sel], px.em[sel]
        w, ew = wo[sel], ewo[sel]
        w2o, ew2o = w * w, 2 * w * ew + ew * ew
        for dx in (0, 1):
            cx = bx[xx] + dx
            wx = (wx1 if dx == 0 else wx2)[xx]
            for dy in (0, 1):
                cy = by[yy] + dy
                wy = (wy1 if dy == 0 else wy2)[yy]
                ok = (cx >= 0) & (cx < cw) & (cy >= 0) & (cy < ch)
                ex, ey = (ewx1 if dx == 0 else ewx2)[xx], (ewy1 if dy == 0 else ewy2)[yy]
                v = m * wx * wy * w2o
                e = (v * 4 * U + em * wx * wy * w2o + m * w2o * (ex * wy + wx * ey + ex * ey)
                     + m * wx * wy * ew2o)
                idx = ((bb * ch + cy) * cw + cx)[ok]
                hist += np.bincount(idx, v[ok], nbin)
                err += np.bincount(idx, e[ok], nbin)
                cnt += np.bincount(idx, None, nbin)
    err += LAMBDA * np.sqrt(cnt) * U * hist
    return hist.reshape(2 * K, ch, cw), err.reshape(2 * K, ch, cw)


def emulate_hist(px, cs, K, defect=None):
    """The kernels' float32 histograms [2K][hogH][hogW] in their vote order (module docstring)."""
    H, W = px.shape
    cw, ch = grid(W, H, cs)
    bx, wx1, wx2 = spatial32(W, cs)
    by, wy1, wy2 = spatial32(H, cs)
    if defect and defect[0] == "swap_w_column":                   # w1 and w2 exchanged for one column
        x = defect[1]
        wx1, wx2 = wx1.copy(), wx2.copy()
        wx1[x], wx2[x] = wx2[x], wx1[x]
    nb = len(px.bins)
    hist = np.zeros((2 * K, ch, cw), f32)
    for ci in range(cw):
        cols = np.nonzero((bx == ci) | (bx == ci - 1))[0]
        if cols.size == 0:
            continue
        x0, x1 = cols[0], cols[-1] + 1
        wxc = np.where(bx[x0:x1] == ci, wx1[x0:x1], wx2[x0:x1]).astype(f32)
        nx = x1 - x0
        c = np.zeros((2 * K, H, nx * nb), f32)                    # per row, per (pixel, orientation entry): the addend
        for j in range(nb):
            b = px.bins[j][:, x0:x1]
            g = px.m32[:, x0:x1]
            if px.bilinear:
                wo = px.wo32[j][:, x0:x1]
                add = ((g * (wxc[None] * wo).astype(f32)).astype(f32) * wo).astype(f32)
            else:
                add = (g * wxc[None]).astype(f32)
            yy, xx = np.nonzero(b >= 0)
            c[b[yy, xx], yy, xx * nb + j] = add[yy, xx]
        T = np.add.accumulate(c, axis=2, dtype=f32)[:, :, -1]     # sequential float32 sum, x ascending
        for cj in range(ch):
            rows = np.nonzero((by == cj) | (by == cj - 1))[0]
            if rows.size == 0:
                continue
            y0, y1 = rows[0], rows[-1] + 1
            wyc = np.where(by[y0:y1] == cj, wy1[y0:y1], wy2[y0:y1]).astype(f32)
            terms = (T[:, y0:y1] * wyc[None]).astype(f32)
            hist[:, cj, ci] = np.add.accumulate(terms, axis=1, dtype=f32)[:, -1]
    return hist


# ---- normalisation and projection --------------------------------------------------------------------------------------------
def _block_index(n):
    """Per cell coordinate: the clamped (lower, upper) neighbours of hog.c:930-933."""
    i = np.arange(n)
    return np.maximum(i - 1, 0), np.minimum(i + 1, n - 1)


def features64(hist, eh, variant, K, stats=None):
    """Float64 features [dd][hogH][hogW] and their bars from float64 histograms and bars.  stats (a dict) receives the number
    of clamped values of haf, hbf and hcf over all cells, bins and factors."""
    _, ch, cw = hist.shape
    Ek = hist[:K] + hist[K:]
    eEk = eh[:K] + eh[K:]
    E = np.sum(Ek ** 2, axis=0)
    eE = np.sum(2 * Ek * eEk + eEk ** 2, axis=0) + (2 * K + 2) * U * E
    xm, xp = _block_index(cw)
    ym, yp = _block_index(ch)
    X = np.arange(cw)[None, :]; Y = np.arange(ch)[:, None]
    fac, efac = [], []
    for q in range(4):
        xa, xb = (X, xp[X]) if q & 1 else (xm[X], X)
        ya, yb = (Y, yp[Y]) if q & 2 else (ym[Y], Y)
        s = E[ya, xa] + E[ya, xb] + E[yb, xa] + E[yb, xb] + 1e-4
        es = eE[ya, xa] + eE[ya, xb] + eE[yb, xa] + eE[yb, xb]
        f = 1.0 / np.sqrt(s)
        fac.append(f)
        efac.append(0.5 * f * es / s + 4 * 2.0 ** -53 * f)

    def clamp(v, e):
        return np.minimum(v, 0.2), np.where(v > 0.2 + e, 0.0, e)

    dd = dims(variant, K)
    out = np.zeros((dd, ch, cw)); err = np.zeros((dd, ch, cw))
    t = np.zeros((4, ch, cw)); et = np.zeros((4, ch, cw))
    for k in range(K):
        ha, hb, ea, eb = hist[k], hist[k + K], eh[k], eh[k + K]
        sa = np.zeros((ch, cw)); sb = np.zeros((ch, cw)); esa = np.zeros((ch, cw)); esb = np.zeros((ch, cw))
        sc = np.zeros((ch, cw)); esc = np.zeros((ch, cw))
        for q in range(4):
            f, ef = fac[q], efac[q]
            haf, ehaf = f * ha, f * ea + ha * ef
            hbf, ehbf = f * hb, f * eb + hb * ef
            if stats is not None:
                for name, val in (("haf", haf), ("hbf", hbf), ("hcf", haf + hbf)):
                    stats[name] = stats.get(name, 0) + int(np.sum(val > 0.2))
            hcf, ehcf = clamp(haf + hbf, ehaf + ehbf)
            haf, ehaf = clamp(haf, ehaf)
            hbf, ehbf = clamp(hbf, ehbf)
            sa += haf; esa += ehaf; sb += hbf; esb += ehbf; sc += hcf; esc += ehcf
            t[q] += hcf; et[q] += ehcf
            if variant == 0:
                out[k + q * K], err[k + q * K] = hcf, ehcf
        if variant == 1:
            out[k], err[k] = 0.5 * sa, 0.5 * esa
            out[k + K], err[k + K] = 0.5 * sb, 0.5 * esb
            out[k + 2 * K], err[k + 2 * K] = 0.5 * sc, 0.5 * esc
    if variant == 1:
        c18 = 1.0 / math.sqrt(18.0)
        for q in range(4):
            out[3 * K + q] = c18 * t[q]
            err[3 * K + q] = c18 * et[q] + 3 * U * c18 * t[q]
    err += 2 * U * np.abs(out)                                   # the float store (u |v|) and the double chain, with room
    return out, err


def features32(hist, variant, K, defect=None, tile=None):
    """hog_cell_energy / hog_cell_factors / hog_cell_features on float32 histograms: the kernels' normalisation, result float32.
    tile: the dense kernel's tile side (only the halo defect needs it)."""
    _, ch, cw = hist.shape
    E = np.zeros((ch, cw), f32)
    for k in range(K):
        h = (hist[k] + hist[k + K]).astype(f32)
        E = (E + (h * h).astype(f32)).astype(f32)
    E = E.astype(np.float64)
    xm, xp = _block_index(cw)
    ym, yp = _block_index(ch)
    if defect and defect[0] == "edge_factor":                     # left edge: neighbour reflected (x + 1) instead of clamped
        xm = xm.copy(); xm[0] = min(1, cw - 1)
    X = np.arange(cw)[None, :]; Y = np.arange(ch)[:, None]
    eps = 0.0 if defect and defect[0] == "no_eps" else 1e-4

    def factors(E):
        fac = []
        for q in range(4):
            xa, xb = (X, xp[X]) if q & 1 else (xm[X], X)
            ya, yb = (Y, yp[Y]) if q & 2 else (ym[Y], Y)
            s = ((E[ya, xa] + E[ya, xb]) + E[yb, xa]) + E[yb, xb]
            with np.errstate(divide="ignore"):
                fac.append(1.0 / np.sqrt(s + eps))
        return fac

    fac = factors(E)
    if defect and defect[0] == "halo_unvoted":                    # the tile at column `tile` sees its left halo column unvoted
        Eh = E.copy()
        Eh[:, tile - 1] = 0.0
        fac = [np.where(X == tile, g, f) for f, g in zip(fac, factors(Eh))]
    clampq = defect[1] if defect and defect[0] == "no_clamp" else None
    dd = dims(variant, K)
    out = np.zeros((dd, ch, cw), f32)
    t = [np.zeros((ch, cw)) for _ in range(4)]
    for k in range(K):
        ha, hb = hist[k].astype(np.float64), hist[k + K].astype(np.float64)
        sa = sb = sc = 0.0
        hcv = []
        for q in range(4):
            with np.errstate(invalid="ignore"):
                haf, hbf = fac[q] * ha, fac[q] * hb
            hcf = haf + hbf
            haf = haf if clampq == "haf" else np.minimum(haf, 0.2)
            hbf = hbf if clampq == "hbf" else np.minimum(hbf, 0.2)
            hcf = hcf if clampq == "hcf" else np.minimum(hcf, 0.2)
            hcv.append(hcf)
            sa, sb, sc = sa + haf, sb + hbf, sc + hcf
            t[q] = t[q] + hcf
        if variant == 1:
            out[k], out[k + K], out[k + 2 * K] = 0.5 * sa, 0.5 * sb, 0.5 * sc
        else:
            for q in range(4):
                out[k + q * K] = hcv[q]
    if variant == 1:
        c18 = float(f32(1) / np.sqrt(f32(18)))
        if defect and defect[0] == "texture3":                    # texture dim 0 sums the clamped sums of three block factors
            t[0] = t[0] + t[1] + t[2]
        for q in range(4):
            out[3 * K + q] = c18 * t[q]
    return out


def truth(px, cs, K, variant, stats=None):
    """Float64 features [dd][hogH][hogW] and their bars."""
    h, e = hist64(px, cs, K)
    return features64(h, e, variant, K, stats)


def emulate(px, cs, K, variant, defect=None, tile=None):
    """The kernels' float32 features in their order, optionally with a planted defect:
      ("drop", y, x)            pixel (y, x) does not vote
      ("bin", y, x, delta)      pixel (y, x) votes into bin b + delta (mod 2K) instead of b
      ("swap_w_column", x)      w1 and w2 exchanged for column x
      ("swap_wo", y, x)         bilinear: w0 and w1 exchanged at pixel (y, x)
      ("edge_factor",)          left-edge block factors from the reflected neighbour
      ("no_eps",)               the 1e-4 of hog_block_factor missing
      ("no_clamp", "haf" | "hbf" | "hcf")
      ("texture3",)             texture dim 0 summing three block factors' clamped sums
      ("halo_unvoted",)         dense: the halo column left of the second tile unvoted (its energy read as 0)"""
    if defect and defect[0] in ("drop", "bin", "swap_wo"):
        y, x = defect[1], defect[2]
        bins = [b.copy() for b in px.bins]
        m32 = px.m32.copy()
        wo32 = [w.copy() for w in px.wo32]
        if defect[0] == "drop":
            m32[y, x] = 0
            for b in bins:
                b[y, x] = -1
        elif defect[0] == "bin":
            K2 = 2 * K
            bins[0][y, x] = (bins[0][y, x] + defect[3]) % K2
        else:
            wo32[0][y, x], wo32[1][y, x] = wo32[1][y, x], wo32[0][y, x]
        px = Pixels(px.m, px.em, m32, bins, px.wo, px.ewo, wo32)
    h = emulate_hist(px, cs, K, defect)
    return features32(h, variant, K, defect, tile)


def ratio(got, want, bar):
    """Per-element |got - want| / bar; a zero bar demands an exact match (inf otherwise, 0 when equal)."""
    got = np.asarray(got, np.float64)
    d = np.abs(got - want)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bar > 0, d / np.where(bar > 0, bar, 1), np.where(d == 0, 0.0, np.inf))
    return np.where(np.isfinite(got), r, np.inf)


def worst(got, want, bar):
    return float(np.max(ratio(got, want, bar))) if np.size(want) else 0.0


# ---- inputs that reach the blind spots ---------------------------------------------------------------------------------------
def blind_spot_frame(H, W, seed, cs=4):
    """An 8-bit frame (values near 128) of +-1 grey-level texture, with a strong step edge crossing a few cells (small features
    next to large ones), a flat block of at least 3 x 3 cells (exact zeros), and a bright saturating square whose edges drive
    many factors past the 0.2 clamp."""
    rng = np.random.default_rng(seed)
    img = 128 + rng.integers(-1, 2, (H, W))
    # strong edge: a vertical step of 120 grey levels over a band of rows in the left part
    ex = max(2, W // 5)
    y0, y1 = H // 5, max(H // 5 + 2, 2 * H // 5)
    img[y0:y1, :ex] += 120
    # flat block in the lower right quadrant: 3 x 3 cells plus a 2-pixel margin where the frame allows
    side = min(3 * cs + 4, max(W // 3, 3), max(H // 3, 3))
    img[H - side:H, W - side:W] = 77
    # bright square in the upper right part
    s = max(3, min(H, W) // 4)
    img[1:1 + s, W - 2 * s - 1:W - s - 1] = 250
    return np.clip(img, 0, 255).astype(np.uint8)


def kinds(feat, bar, stats):
    """What an input reached: 'flat' cells (every feature and bar exactly 0), 'small' features (non-zero, below 1e-2 of the
    largest), and clamped haf / hbf / hcf values (stats of features64)."""
    flat = np.all(feat == 0, axis=0) & np.all(bar == 0, axis=0)
    small = (feat > 0) & (feat < 1e-2 * np.max(feat))
    return {"flat": int(np.sum(flat)), "small": int(np.sum(small)), **{k: stats.get(k, 0) for k in ("haf", "hbf", "hcf")}}


def _repair(frame, bad, rng, amp):
    """Move the right-hand or the lower neighbour (at random) of every pixel whose decision is in doubt: its gradient changes,
    its own value does not."""
    yy, xx = np.nonzero(bad)
    right = rng.random(yy.size) < 0.5
    xx = np.where(right, np.minimum(xx + 1, frame.shape[-1] - 1), xx)
    yy = np.where(right, yy, np.minimum(yy + 1, frame.shape[-2] - 1))
    noise = rng.uniform(-amp, amp, (frame.shape[0], yy.size)).astype(f32)
    frame[:, yy, xx] = np.clip(frame[:, yy, xx] + noise, 0, None)
    return frame


def decided_float_frame(frame, K, bilinear, seed=0, amp=0.25, tries=200):
    """A float32 (C, H, W) frame close to `frame` whose every orientation and channel decision has its float64 margin (pixels in
    doubt get their right-hand neighbour moved, until none is left)."""
    frame = np.array(frame, f32, copy=True)
    if frame.ndim == 2:
        frame = frame[None]
    rng = np.random.default_rng(seed)
    for _ in range(tries):
        bad = decision_doubt(frame, K, bilinear)
        if not bad.any():
            return frame
        frame = _repair(frame, bad, rng, amp)
    raise AssertionError("could not move the frame's decisions out of the float32 margin")


def polar_field(H, W, seed, K, directed, bilinear, decades=6):
    """A modulus field over `decades` orders of magnitude (log-uniform from 1e-3), with a zero band and negative moduli (which
    do not vote), and float32 angles whose ho = angle / (pi / K) keeps the float64 margin from every bin decision; some angles
    are negative or beyond 2 pi."""
    rng = np.random.default_rng(seed)
    m = (10.0 ** rng.uniform(-3, -3 + decades, (H, W))).astype(f32)
    m[H // 2, :] = 0
    m[:, W // 3] = -1
    period = 2 * K if directed else K
    ang = np.zeros((H, W), f32)
    todo = np.ones((H, W), bool)
    for _ in range(100):
        ho = rng.integers(-period, 2 * period, (H, W)) + rng.uniform(0.02, 0.98, (H, W))
        a = (ho * math.pi / K).astype(f32)
        ang = np.where(todo, a, ang)
        hv = ang.astype(np.float64) / (math.pi / K)
        frac = hv - np.floor(hv)
        e = MARGIN * U * (np.abs(hv) + 2)
        ok = (frac > e) & (frac < 1 - e) & (np.abs(frac - 0.5) > e) & (np.floor(hv) == np.floor((hv).astype(f32)))
        todo = ~ok
        if not todo.any():
            return m, ang.astype(f32)
    raise AssertionError("could not place the angles")


def float_case_frame(C, H, W, seed, cs, K, bil, scale=1.0):
    """A float32 (C, H, W) blind-spot frame (values in [0, 255] times scale) with +-0.3 noise and a flat block, whose decisions
    all keep their float64 margin."""
    base = np.stack([blind_spot_frame(H, W, seed=seed + c, cs=cs) for c in range(C)]).astype(f32)
    base += np.random.default_rng(seed).uniform(-0.3, 0.3, base.shape).astype(f32)
    side = min(3 * cs + 4, H // 3, W // 3)
    base[:, H - side:, W - side:] = 77.0
    return decided_float_frame((base * f32(scale)).astype(f32), K, bil, seed=seed, amp=0.25 * scale)


# the image frames of the sd_hog_dense_images tests: (channels, layout, cs, K, H, W, scale of the float frames)
IMAGE_CASES = [
    (1, "planar", 4, 4, 61, 83, 1.0), (1, "planar", 8, 9, 75, 101, 1 / 255), (3, "planar", 4, 9, 61, 83, 1.0),
    (3, "interleaved", 6, 4, 67, 59, 1 / 255), (3, "planar", 1, 2, 30, 34, 1.0), (16, "planar", 5, 16, 47, 53, 1.0),
    (16, "interleaved", 11, 1, 70, 66, 1.0), (3, "planar", 32, 16, 100, 90, 1.0),
]


def image_case_frame(case, kind, bil):
    """The planar (C, H, W) frame of an IMAGE_CASES entry: 'f32' (float_case_frame) or 'u8' (blind-spot planes, channel c's
    contrast scaled by (c + 1) / 2 so that the channels' gradients differ)."""
    C, layout, cs, K, H, W, scale = case
    if kind == "f32":
        return float_case_frame(C, H, W, cs * 31 + K, cs, K, bil, scale)
    f = np.stack([blind_spot_frame(H, W, seed=cs + c, cs=cs) for c in range(C)])
    if C > 1:
        f = np.stack([np.clip(128 + (f[c].astype(int) - 128) * (c + 1) // 2 + c, 0, 255) for c in range(C)]).astype(np.uint8)
    return f

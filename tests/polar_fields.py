"""Gradient fields and the angle-to-bin rule of vl_hog_put_polar_field (hog.c:784-800) for the polar dense-HOG tests.

polar_bins is a numpy float32 restatement of the rule the device applies (polar_bins in csrc/sd_hog_dense.cu): the Euclidean
residue of floor(ho) computed without hog.c's loop.  tests/test_vl_hog_polar_oracle.py pins it to hog.c."""
import numpy as np

VL_PI = 3.141592653589793     # hog.h's VL_PI, the same double as np.pi


def polar_ho(angle, K):
    """ho = (float)((double)angle / (VL_PI / K)), as hog.c:784 rounds it."""
    return (np.asarray(angle, dtype=np.float32).astype(np.float64) / (VL_PI / K)).astype(np.float32)


def polar_bins(angle, K, directed):
    """(nearest bin, bilinear first bin, bilinear second bin, second weight wo2) of float32 angles; bins are -1 where ho is not
    finite.  Nearest: bino + 1 unless wo1 > wo2 (a tie goes to bino + 1); all bins modulo K, or 2K when directed."""
    period = np.float32(2 * K if directed else K)
    with np.errstate(invalid="ignore", over="ignore"):
        ho = polar_ho(angle, K)
        ok = np.isfinite(ho)
        bino = np.floor(np.where(ok, ho, np.float32(0)))
        wo2 = (np.where(ok, ho, np.float32(0)) - bino).astype(np.float32)
        wo1 = (np.float32(1) - wo2).astype(np.float32)
        r = np.fmod(bino, period)
        r = np.where(r < 0, r + period, r).astype(np.int64)
    p = int(period)
    b1 = (r + 1) % p
    near = np.where(wo1 > wo2, r, b1)
    return (np.where(ok, near, -1), np.where(ok, r, -1), np.where(ok, b1, -1), np.where(ok, wo2, np.float32(0)))


def half_steps(K, lo=-2, hi=2):
    """Float32 angles at (b + 0.5) pi / K for b in [lo K, hi K) whose ho is exactly b + 0.5 (a few ulps of search each);
    returns (angles, number of half steps tried)."""
    out, tried = [], 0
    for b in range(lo * K, hi * K):
        tried += 1
        target = np.float32(b + 0.5)
        t = np.float32((b + 0.5) * VL_PI / K)
        for _ in range(16):
            ho = polar_ho(t, K)
            if ho == target:
                out.append(t)
                break
            t = np.nextafter(t, np.float32(np.inf) if ho < target else np.float32(-np.inf), dtype=np.float32)
    return np.array(out, dtype=np.float32), tried


def angle_sweep(K):
    """Exact half steps (ties), exact multiples of the step, large magnitudes and negative angles."""
    halves, _ = half_steps(K)
    multiples = np.array([b * VL_PI / K for b in range(-2 * K, 2 * K + 1)], dtype=np.float32)
    large = np.array([1e4, -1e4, 1e7, -1e7, 12345.678, -98765.43, 3e5 + 0.25, -7e6 - 0.5], dtype=np.float32)
    rng = np.random.default_rng(K)
    negative = -rng.uniform(0, 6 * np.pi, 8).astype(np.float32)
    return np.concatenate([halves, multiples, large, negative])


def smooth_field(h, w, seed):
    """(modulus, angle): smooth structure plus noise; moduli with zeros and negatives, angles spread over [-4 pi, 4 pi]."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    m = 1.0 + np.sin(x / (7.0 + seed % 5) + np.cos(y / 13.0)) + rng.normal(0, 0.3, (h, w))
    m[rng.random((h, w)) < 0.05] = 0.0
    a = 4 * np.pi * np.sin(x / 23.0 + y / (11.0 + seed % 3)) + rng.normal(0, 0.5, (h, w))
    a = np.clip(a, -4 * np.pi, 4 * np.pi)
    return m.astype(np.float32), a.astype(np.float32)


def one_vote_per_cell(h, w, cs, angles, seed):
    """(modulus, angle): exactly one pixel per cell (a pseudo-random one inside the cell) has a non-zero modulus, and its angle
    is the next of `angles` (cycled)."""
    rng = np.random.default_rng(seed)
    m = np.zeros((h, w), np.float32)
    a = np.zeros((h, w), np.float32)
    i = 0
    for y0 in range(0, h, cs):
        for x0 in range(0, w, cs):
            y = y0 + rng.integers(0, min(cs, h - y0))
            x = x0 + rng.integers(0, min(cs, w - x0))
            m[y, x] = np.float32(rng.uniform(0.5, 2.0))
            a[y, x] = angles[i % len(angles)]
            i += 1
    return m, a

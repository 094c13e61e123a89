"""A numpy restatement of sd_hog_distance_transform_exact (include/sd_b200.h): per line, the float64 lower envelope of the finite
scores in the header's operation order, the values fl(f(q*) - c(q* - p)) in float32, pass X along rows and then pass Y along
columns of pass X's output.  Every line of a pass is walked at once, position by position, so that each float64 operation is
the one the kernel makes: numpy's float64 arithmetic rounds each operation and fuses none."""
import numpy as np


def cost(a, b, d):
    """c(d) = (float)(((double) a d) d + (double) b d), the bounded call's cost-table formula, for int64 displacements d."""
    x = np.asarray(d, np.int64).astype(np.float64)
    return (a * x * x + b * x).astype(np.float32)


def meet(q, fq, r, fr, a, b):
    """s(q, r) of the header: the point past which r owns against q (arrays of equal shape; r > q)."""
    dq = (r - q).astype(np.float64)
    sq = ((r - q).astype(np.int64) * (r + q).astype(np.int64)).astype(np.float64)
    num = ((fq.astype(np.float64) - fr.astype(np.float64)) + a * sq) + b * dq
    return num / ((a + a) * dq)


def lines(f, a, b):
    """f (L, n) float32 lines sharing weights (a, b) -> (values (L, n) float32, owner (L, n) int64, -1 where the line has no
    candidate)."""
    f = np.asarray(f, np.float32)
    L, n = f.shape
    a, b = float(np.float32(a)), float(np.float32(b))
    z = np.zeros((L, n))
    v = np.zeros((L, n), np.int64)
    fv = np.zeros((L, n), np.float32)
    cnt = np.zeros(L, np.int64)
    rows = np.arange(L)
    with np.errstate(over="ignore", invalid="ignore"):
        for q in range(n):
            fq = f[:, q]
            act = np.isfinite(fq)
            s = np.full(L, -np.inf)
            # pop while the top's z is not below the meeting point; lines stop popping independently
            check = act & (cnt > 0)
            while check.any():
                i = rows[check]
                top = cnt[i] - 1
                si = meet(v[i, top], fv[i, top], np.full(len(i), q), fq[i], a, b)
                keep = si > z[i, top]
                s[i[keep]] = si[keep]
                pop = i[~keep]
                cnt[pop] -= 1
                s[pop] = -np.inf
                check = np.zeros(L, bool)
                check[pop] = cnt[pop] > 0
            i = rows[act]
            z[i, cnt[i]] = s[i]
            v[i, cnt[i]] = q
            fv[i, cnt[i]] = fq[i]
            cnt[i] += 1
        values = np.full((L, n), -np.inf, np.float32)
        owner = np.full((L, n), -1, np.int64)
        e = np.zeros(L, np.int64)
        has = cnt > 0
        for p in range(n):
            move = has & (e + 1 < cnt)
            while move.any():
                i = rows[move]
                step = z[i, e[i] + 1] < p
                e[i[step]] += 1
                move = np.zeros(L, bool)
                move[i[step]] = e[i[step]] + 1 < cnt[i[step]]
            i = rows[has]
            q = v[i, e[i]]
            owner[i, p] = q
            values[i, p] = fv[i, e[i]] - cost(a, b, q - p)
    return values, owner


def transform(s, w):
    """One plane: s (h, w) float32, w = (w0, w1, w2, w3) -> (D (h, w) float32, placements (h, w, 2) int32 of (u, v), (-1, -1)
    for none)."""
    s = np.asarray(s, np.float32)
    w = np.asarray(w, np.float32)
    t, ox = lines(s, w[0], w[1])
    Dt, oy = lines(t.T, w[2], w[3])
    D, vy = Dt.T, oy.T
    place = np.full(s.shape + (2,), -1, np.int32)
    vv, uu = np.nonzero(vy >= 0)
    place[vv, uu, 0] = ox[vy[vv, uu], uu]
    place[vv, uu, 1] = vy[vv, uu]
    return np.ascontiguousarray(D), place


def brute_line(f, a, b):
    """float64 objective of every (position p, candidate q) of one line: f(q) - (a d^2 + b d), d = q - p, in float64 (-inf for
    a non-finite f(q)) -> (n, n)."""
    f = np.asarray(f, np.float32).astype(np.float64)
    a, b = float(np.float32(a)), float(np.float32(b))
    n = len(f)
    d = np.arange(n)[None, :] - np.arange(n)[:, None]
    obj = f[None, :] - (a * d * d + b * d)
    return np.where(np.isfinite(f)[None, :], obj, -np.inf)

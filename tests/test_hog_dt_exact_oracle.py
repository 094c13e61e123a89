"""The numpy restatement of the exact transform (hog_dt_exact_ref.py) against independent rules, on the CPU.

- Per line, against a float64 brute force over every candidate: each owner maximises the float64 objective f(q) - c64(q - p)
  to within its rounding, is the first maximiser wherever the best and second best candidates are apart by more than that, and
  every value is fl(f(q*) - c(q* - p)).  Lines mix NaN and +-inf with finite scores, and weights reach from tiny w0 (a score
  pulls across the whole line) to large asymmetric w1.
- On small integers, where every operation is exact, the owners are the first exact maximisers, and the 2-D transform equals
  hog_parts_ref.py's bounded rule at R >= max(w, h) bit for bit, placements included."""
import numpy as np
import pytest

import hog_dt_exact_ref as ex
import hog_parts_ref as ref


def _check_lines(f, a, b, exact):
    vals, owner = ex.lines(f, a, b)
    for i in range(f.shape[0]):
        obj = ex.brute_line(f[i], a, b)
        finite = np.isfinite(f[i])
        if not finite.any():
            assert np.all(owner[i] == -1) and np.all(np.isneginf(vals[i]))
            continue
        best = obj.max(axis=1)
        p = np.arange(f.shape[1])
        got = obj[p, owner[i]]
        assert np.all(finite[owner[i]])
        scale = np.abs(obj[:, finite]).max(axis=1) + 1.0
        tol = 0.0 if exact else 1e-12 * scale
        assert np.all(got >= best - tol), i
        srt = np.concatenate([np.full((len(p), 1), -np.inf), np.sort(obj, axis=1)], axis=1)
        clear = np.full(len(p), True) if exact else srt[:, -1] - srt[:, -2] > tol
        assert np.array_equal(owner[i][clear], np.argmax(obj, axis=1)[clear]), i
        c = ex.cost(np.float64(np.float32(a)), np.float64(np.float32(b)), owner[i] - p)
        assert np.array_equal(vals[i].view(np.int32), (f[i][owner[i]] - c).view(np.int32)), i


@pytest.mark.parametrize("a,b", [(0.05, 0.0), (0.3, -0.2), (1e-6, 0.0), (1e-6, 1e-4), (0.01, 5.0), (2.0, -7.5), (40.0, 3.0)])
def test_lines_against_float64_brute_force(a, b):
    rng = np.random.default_rng(int(a * 1000) + int(abs(b) * 10))
    f = rng.normal(0, 3, (40, 73)).astype(np.float32)
    flat = f.reshape(-1)
    idx = rng.choice(flat.size, flat.size // 8, replace=False)
    flat[idx[0::3]] = np.nan
    flat[idx[1::3]] = np.inf
    flat[idx[2::3]] = -np.inf
    f[3] = np.nan                                              # no candidate
    f[4, :] = -np.inf
    f[4, 17] = 1.0                                             # one candidate
    f[5, :] = 2.5                                              # constant: ties everywhere when b = 0
    _check_lines(f, a, b, exact=False)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 200])
def test_integer_lines_take_the_first_exact_maximiser(n):
    rng = np.random.default_rng(n)
    for a in (1, 2, 3):
        for b in (-4, -1, 0, 1, 5):
            f = rng.integers(-12, 13, (25, n)).astype(np.float32)
            f[0] = 0.0
            _check_lines(f, a, b, exact=True)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 9), (9, 1), (7, 12), (20, 33), (33, 5)])
def test_integer_maps_equal_the_bounded_rule_at_full_reach(h, w):
    rng = np.random.default_rng(h * 100 + w)
    R = max(h, w)
    for _ in range(4):
        s = rng.integers(-20, 21, (h, w)).astype(np.float32)
        d = np.array([rng.integers(1, 4), rng.integers(-5, 6), rng.integers(1, 4), rng.integers(-5, 6)], np.float32)
        D, pl = ex.transform(s, d)
        Db, plb = ref.transform(s, d, R)
        assert np.array_equal(D.view(np.int32), Db.view(np.int32))
        assert np.array_equal(pl, plb)


def test_placements_follow_the_owners_of_both_passes():
    rng = np.random.default_rng(3)
    s = rng.normal(0, 2, (23, 41)).astype(np.float32)
    s[5] = np.nan                                              # a row without candidates
    s[:, 7] = -np.inf
    d = np.array([0.02, 0.3, 0.05, -0.4], np.float32)
    D, pl = ex.transform(s, d)
    t, ox = ex.lines(s, d[0], d[1])
    _, oy = ex.lines(t.T, d[2], d[3])
    for v in range(s.shape[0]):
        for u in range(s.shape[1]):
            vs = oy[u, v]
            assert tuple(pl[v, u]) == ((ox[vs, u], vs) if vs >= 0 else (-1, -1))
            assert vs != 5

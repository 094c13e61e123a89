"""The chunked training level (sd_train_level) restated in numpy: no GPU needed.

A level's rows arrive in chunks.  The first chunk's column means are the pilot shift p; every chunk is shifted by p before
its [A' | b] enters the accumulated Gram.  The solve then works from the shifted Gram exactly as solve_gram_impl does:
  - ||A^T A||_F of the UNshifted matrix is rebuilt entry by entry from G', its bias column s' and p (frob_upper_centred_kernel),
    and gives the MatrixNorm lambda (regressors.hpp:126-148);
  - the bias column is eliminated first (bias_downdate_kernel): G'' = G' - s' s'^T / n, the exact centring of any shifted Gram;
  - the bias is shifted back (bias_finish_kernel): c = c' - p.w.
In float64 this is the direct solve for every chunking; accumulated in float32 the pilot keeps the digits that exact centring
keeps, and the unshifted Gram loses them (DESIGN 4.3)."""
import numpy as np
import pytest


def _features(n, D, seed):
    """HOG-like rows: non-negative, clamped (mean well above the spread), last column all ones."""
    rng = np.random.default_rng(seed)
    A = (0.12 + np.minimum(np.abs(rng.standard_normal((n, D))) * 0.03, 0.1)).astype(np.float32)
    A[:, ::5] *= 0.5
    A[:, -1] = 1.0
    W = rng.standard_normal((D, 6)) * 0.3
    B = (A.astype(np.float64) @ W + 0.05 * rng.standard_normal((n, 6))).astype(np.float32)
    return A, B


def _lambda(fro, n, param):
    return param * fro / n


def _direct(A, B, param):
    """regressors.hpp:199-234 in float64: X = (A^T A + Lambda)^-1 A^T B, bias row unregularised."""
    A64, B64 = A.astype(np.float64), B.astype(np.float64)
    G = A64.T @ A64
    lam = _lambda(np.linalg.norm(G), A.shape[0], param)
    reg = np.eye(G.shape[0]) * lam
    reg[-1, -1] = 0.0
    return np.linalg.solve(G + reg, A64.T @ B64), lam


def _chunked(A, B, param, chunk, dtype, shift="pilot"):
    """sd_train_level's algorithm; the Gram is accumulated in `dtype`, everything after it in float64."""
    n, D = A.shape
    if shift == "pilot":
        p = A[:chunk].astype(np.float64).mean(axis=0)
    elif shift == "exact":
        p = A.astype(np.float64).mean(axis=0)
    else:
        p = np.zeros(D)
    p[-1] = 0.0                                                     # the bias column is never shifted
    p = p.astype(np.float32).astype(np.float64)                     # the device holds the shift in float32
    G = np.zeros((D, D), dtype=dtype)
    R = np.zeros((D, B.shape[1]), dtype=dtype)
    for r0 in range(0, n, chunk):
        Ac = (A[r0:r0 + chunk].astype(dtype) - p.astype(dtype)).astype(dtype)
        G += Ac.T @ Ac
        R += Ac.T @ B[r0:r0 + chunk].astype(dtype)
    G, R = G.astype(np.float64), R.astype(np.float64)
    s = G[:, -1]                                                    # s' = A'^T 1; s'[-1] = n
    nn = s[-1]
    # ||A^T A||_F from the shifted Gram: A^T A = G' + s' p^T + p s'^T + n p p^T
    fro = np.linalg.norm(G + np.outer(s, p) + np.outer(p, s) + nn * np.outer(p, p))
    lam = _lambda(fro, n, param)
    H = G[:-1, :-1] + lam * np.eye(D - 1)
    # bias column first: c' = (r_b - s'^T w) / n, (H - s' s'^T / n) w = R' - s' r_b / n
    sf, rb = s[:-1], R[-1]
    w = np.linalg.solve(H - np.outer(sf, sf) / nn, R[:-1] - np.outer(sf, rb) / nn)
    c = (rb - sf @ w) / nn - p[:-1] @ w                             # shifted back: c = c' - p.w
    return np.vstack([w, c[None, :]]), lam


def _rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


@pytest.mark.parametrize("chunk", [900, 300, 301, 899], ids=["one", "thirds", "ragged", "last-one-row"])
def test_float64_chunked_solve_is_the_direct_solve(chunk):
    A, B = _features(900, 120, seed=3)
    X, lam = _direct(A, B, 1.5)
    Xc, lamc = _chunked(A, B, 1.5, chunk, np.float64)
    assert abs(lamc - lam) <= 1e-12 * lam
    assert _rel(Xc, X) <= 1e-10


def test_pilot_shift_keeps_the_digits_of_exact_centring():
    A, B = _features(3000, 200, seed=5)
    X64, _ = _direct(A, B, 0.05)
    e_pilot = _rel(_chunked(A, B, 0.05, 500, np.float32, "pilot")[0], X64)
    e_exact = _rel(_chunked(A, B, 0.05, 3000, np.float32, "exact")[0], X64)
    e_raw = _rel(_chunked(A, B, 0.05, 500, np.float32, "none")[0], X64)
    print(f"float32 Gram vs float64 weights: pilot {e_pilot:.2e}, exact mean {e_exact:.2e}, unshifted {e_raw:.2e}")
    assert e_pilot <= 2.0 * e_exact
    assert e_raw >= 100.0 * e_pilot

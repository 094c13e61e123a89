"""The per-element error bars of tests/gemm_ref.py against a numpy restatement of the tensor-core Gram arithmetic (no GPU):
the bars must accept the kernel's arithmetic with margin, at any number of samples, and reject the defects a broken kernel
would show."""
import numpy as np
import pytest

import gemm_ref as R


def _hog_like(rng, n, d):
    """non-negative, bounded, correlated columns and a bias column of ones: every product has the same sign, so a one-signed
    error does not cancel"""
    base = rng.random((n, 4)).astype(np.float32)
    A = np.clip(0.05 * base @ rng.random((4, d)).astype(np.float32) + 0.1 * rng.random((n, d)).astype(np.float32), 0, 0.4)
    A = A.astype(np.float32)
    A[:, -1] = 1.0
    return A


@pytest.mark.parametrize("n,d,m", [(1, 5, 2), (127, 20, 3), (300, 20, 3), (1000, 33, 5), (100_000, 6, 2)])
@pytest.mark.parametrize("unbiased", [False, True])
def test_bar_accepts_the_kernel_arithmetic(n, d, m, unbiased):
    rng = np.random.default_rng(n + d)
    A = _hog_like(rng, n, d)
    B = (0.05 * rng.standard_normal((n, m))).astype(np.float32)
    mode = 3 if unbiased else 0
    G = R.emulate_gram(A, B, unbiased=unbiased)
    excess, _ = R.gram_excess(G, A, B, mode)
    print(f"n={n} mode={mode}: error / bar {excess:.3f} (tau {R.tau_gram(mode, n):.2e})")
    assert excess <= 0.5


def test_bar_rejects_defects():
    rng = np.random.default_rng(5)
    n, d, m = 300, 20, 3
    A = _hog_like(rng, n, d)
    B = (0.05 * rng.standard_normal((n, m))).astype(np.float32)
    ok, _ = R.gram_excess(R.emulate_gram(A, B), A, B, 0)
    assert ok <= 0.5
    dropped_sample, _ = R.gram_excess(R.emulate_gram(A[:-1], B[:-1]), A, B, 0)
    A_col = A.copy()
    A_col[:, 7] = 0.0
    dropped_column, _ = R.gram_excess(R.emulate_gram(A_col, B), A, B, 0)
    G_rhs = R.emulate_gram(A, B)
    G_rhs[:, d + m - 1] = 0.0
    dropped_rhs, _ = R.gram_excess(G_rhs, A, B, 0)
    dropped_lohi, _ = R.gram_excess(R.emulate_gram(A, B, drop_lohi=True), A, B, 0)
    print(f"error / bar: exact arithmetic {ok:.2f}, one sample dropped {dropped_sample:.1f}, one column dropped {dropped_column:.1f}, "
          f"one right-hand side dropped {dropped_rhs:.1f}, lo*hi dropped {dropped_lohi:.1f}")
    for e in (dropped_sample, dropped_column, dropped_rhs, dropped_lohi):
        assert e > 4.0


def test_single_pass_defect_is_outside_the_3xtf32_bar():
    """a 3xTF32 launch that ran a single TF32 pass (mode 1 arithmetic) must fail the mode-0 bar, and pass its own"""
    rng = np.random.default_rng(8)
    A = _hog_like(rng, 500, 16)
    S = R.trunc_tf32(A)
    G1 = (S.astype(np.float64).T @ S.astype(np.float64)).astype(np.float32)
    assert R.gram_excess(G1, A, None, 0)[0] > 4.0
    assert R.gram_excess(G1, A, None, 1)[0] <= 0.5


def test_predict_bar():
    """the predict bar accepts fp32 chunk sums folded in double, and rejects a missing chunk of the contraction"""
    rng = np.random.default_rng(2)
    A = rng.standard_normal((50, 1000)).astype(np.float32)
    X = rng.standard_normal((1000, 7)).astype(np.float32)
    ref, bar = R.predict_ref(A, X)
    chunks = [np.cumsum(A[:, k:k + 32, None] * X[None, k:k + 32, :], axis=1, dtype=np.float32)[:, -1] for k in range(0, 1000, 32)]
    Y = np.sum(np.stack(chunks).astype(np.float64), axis=0).astype(np.float32)
    assert np.max(np.abs(Y - ref) / bar) <= 0.5
    Y_short = np.sum(np.stack(chunks[:-1]).astype(np.float64), axis=0).astype(np.float32)
    assert np.max(np.abs(Y_short - ref) / bar) > 4.0

"""The per-element bars of tests/chol_ref.py against numpy restatements of the solve (no GPU): the bars must accept the
kernels' arithmetic with margin on every shape of the GPU sweep with D <= 2049 at condition numbers 1e1 to 1e7, and reject
the defects a broken factorisation, elimination or regulariser would show.  The LU restatement is pinned to the oracle."""
import numpy as np
import pytest

import chol_ref as C
import gemm_ref as R

ARITH = {0: "split", 3: "split", 2: "fp32"}


def _shapes():
    """(D, largest M, arithmetic) of the sweep cases with D <= 2049 that have a bar (gram mode 1 has the eta check only)"""
    out = {}
    for D, M, _, mode, _, _, _ in C.SWEEP:
        if D <= 2049 and mode in ARITH:
            key = (D, ARITH[mode])
            out[key] = max(out.get(key, 0), M)
    return [(D, M, a) for (D, a), M in sorted(out.items())]


def test_sweep_reaches_the_tensor_cores():
    """every gram mode that has them (0, 1, 3) runs tensor-core head AND tail updates at every condition number of the sweep,
    every D = 4097 case runs them, and the "skew" / "odd" pitches and gram mode 2 stay on the SIMT route"""
    covered = set()
    for c in C.SWEEP:
        D, M, cond, mode, kind, _, _ = c
        routes = C.case_routes(c)
        if any(tc and tail for tc, tail in routes):
            covered.add((mode, cond))
        if D == 4097:
            assert routes[0] == (True, True), C.sweep_id(c)
        if kind in ("skew", "odd") or mode == 2:
            assert not any(tc for tc, _ in routes), C.sweep_id(c)
        print(C.sweep_id(c), "tensor-core / SIMT SYRK launches", C.syrk_launches(routes))
    for mode in (0, 1, 3):
        for cond in (1e1, 1e3, 1e5, 1e7):
            assert (mode, cond) in covered, (mode, cond)


def _check(G, M, reg, arith, mode, T=None, **kw):
    """worst error / bar of the restated solve of G (w rows and the bias row), or inf when a defect broke positive definiteness;
    T: the float64 truth of G, when it is already known"""
    if T is None:
        T = C.Truth(C.regularise(G, float(np.float32(reg[1])), bool(reg[2])), M)
    try:
        X, _, _ = C.solve_gram_restated(G, M, reg, C.N_DESIGN, arith, **kw)
    except np.linalg.LinAlgError:
        return float("inf"), T, None
    bw = T.bar_w(mode)
    r = max(C.ratio(X[:-1], T.w, bw).max(), float(np.max(np.abs(X[-1] - T.xb) / T.bar_xb(bw))))
    return r, T, X


@pytest.mark.parametrize("D,M,arith", _shapes(), ids=lambda v: str(v))
def test_bars_accept_the_restated_solve(D, M, arith):
    mode = 2 if arith == "fp32" else 0
    for cond in (1e1, 1e3, 1e5, 1e7):
        G = C.designed_gram(D, M, cond, C.LAMBDA_DESIGN, False, seed=D * 1000 + M)
        r, T, X = _check(G, M, (0, C.LAMBDA_DESIGN, 0), arith, mode)
        eta, eta_ref = T.eta(X[:-1]).max(), T.eta_spotrs().max()
        print(f"D={D} M={M} {arith} cond {cond:.0e}: error / bar {r:.4f}, eta {eta:.2e} (spotrs {eta_ref:.2e}, allowed excess "
              f"{T.eta_excess(mode):.2e})")
        assert r <= 0.25
        assert eta <= eta_ref + T.eta_excess(mode)


def test_bars_reject_defects():
    D, M = 1025, 63
    G = C.designed_gram(D, M, 1e1, C.LAMBDA_DESIGN, False, seed=7)
    reg = (0, C.LAMBDA_DESIGN, 0)
    ok, T, _ = _check(G, M, reg, "split", 0)
    got = {}
    for name, kw in [("head tile", dict(defect=("head", 1, 64, 128))),          # panel 1: rows 512.. of the matrix
                     ("tail tile", dict(defect=("tail", 0, 64, 320))),
                     ("fused A^T P row", dict(defect=("fused_row", 1))),
                     ("W for W^T in the back substitution", dict(defect=("backsub_w", 3))),
                     ("bias pivot p - 1", dict(defect=("pivot_n_minus_1",)))]:
        got[name] = _check(G, M, reg, "split", 0, T, **kw)[0]
    got["single-pass TF32 updates"] = _check(G, M, reg, "single", 0, T)[0]
    # the pivot matters as much as the bias column's coupling: a system whose s s^T / p is the size of S
    Gc = C.designed_gram(D, M, 1e1, C.LAMBDA_DESIGN, False, seed=8, coupling=1.0)
    ok_c, Tc, _ = _check(Gc, M, reg, "split", 0)
    assert ok_c <= 0.25
    got["bias pivot p - 1, coupled"] = _check(Gc, M, reg, "split", 0, Tc, defect=("pivot_n_minus_1",))[0]
    print(f"error / bar: correct {ok:.4f}; " + "; ".join(f"{k} {v:.1f}" for k, v in got.items()))
    assert ok <= 0.25
    for name in ("head tile", "tail tile", "fused A^T P row", "W for W^T in the back substitution", "single-pass TF32 updates",
                 "bias pivot p - 1, coupled"):
        assert got[name] > 4.0, name


def _hog_like(rng, n, d):
    base = rng.random((n, 8)).astype(np.float32)
    A = np.clip(0.05 * (base @ rng.random((8, d)).astype(np.float32)) + 0.1 * rng.random((n, d)).astype(np.float32), 0, 0.4)
    A = A.astype(np.float32)
    A[:, -1] = 1.0
    return A


def test_learn_bars_accept_the_restated_learn_and_reject_the_centred_norm():
    """sd_centre_features + sd_learn_centred restated (float32 Gram of the centred rows): the learn bar accepts it, lambda is
    within its bar of the float64 norm of the uncentred A^T A, and a lambda taken from the centred norm is rejected"""
    rng = np.random.default_rng(3)
    N, D, M = 900, 300, 20
    A = _hog_like(rng, N, D)
    B = (0.05 * rng.standard_normal((N, M))).astype(np.float32)
    mu, Ac = C.centre_restated(A, False)
    assert mu[:-1].all() and mu[-1] == 0
    Gc = np.hstack([Ac.T @ Ac, Ac.T @ B]).astype(np.float32)
    reg = (1, 1.5, 0)
    X, Xc, lam = C.solve_gram_restated(Gc, M, reg, N, "split", mu=mu)
    lam_true = 1.5 * np.linalg.norm(R.gram_ref(A)) / N
    assert abs(lam - lam_true) <= C.lambda_bar(A, Ac, mu, 1.5)
    T = C.learn_truth(Ac, B, lam, False)
    bw = T.bar_w(0)
    ok = C.ratio(Xc[:-1], T.w, bw).max()
    Xd, _, lam_c = C.solve_gram_restated(Gc, M, reg, N, "split", mu=mu, defect=("centred_norm",))
    bad = C.ratio(Xd[:-1], T.w, bw).max()
    print(f"lambda {lam:.6g} (float64 {lam_true:.6g}, centred norm {lam_c:.6g}); error / bar {ok:.4f}, centred-norm lambda {bad:.1f}")
    assert ok <= 0.25
    assert bad > 4.0


@pytest.mark.parametrize("D", [20, 100, 256])
def test_lu_restatement_is_the_oracle_solver(oracle, D):
    """lu_restated on the oracle's own float32 Gram, lambda and A^T B gives orc_solve's (precision 0) X bit for bit"""
    rng = np.random.default_rng(D)
    N, M = 300, 6
    A = rng.standard_normal((N, D)).astype(np.float32)
    B = rng.standard_normal((N, M)).astype(np.float32)
    for typ, param, last in [(0, 0.5, 0), (1, 2.0, 1), (0, 0.0, 1)]:
        reg = oracle.Regulariser(typ, param, last)
        Xo, lam = oracle.solve(A, B, reg, 0)
        AtA = oracle.gram(A, 0)
        assert lam == oracle.regulariser_lambda(reg, AtA, N)
        Rh = np.zeros((D, M), np.float32)
        for n in range(N):                                  # A^T B as orc_solve sums it: sample by sample, float32
            Rh = (Rh + (A[n][:, None] * B[n][None, :]).astype(np.float32)).astype(np.float32)
        G = C.regularise(np.hstack([AtA, Rh]), lam, bool(last))
        X, singular = C.lu_restated(G, M)
        assert not singular
        assert np.array_equal(X.view(np.uint32), Xo.view(np.uint32)), f"D={D} reg {(typ, param, last)}"

"""sd_solve_gram, sd_centre_features + sd_learn_centred and LinearRegressor.learn against float64 with the per-element bars of
chol_ref.py: the blocked Cholesky across its block, panel and right-hand-side group edges at condition numbers 1e1 to 1e7, every
gram mode, tight, odd and padded misaligned pitches, both regularisers, a poisoned lower triangle; the learn path with its
centring fallbacks; and the small partial-pivot LU bit for bit against its restatement."""
import ctypes as C

import numpy as np
import pytest

import chol_ref as CR
import gemm_ref as R

pytestmark = pytest.mark.gpu
SD_ERR_NUMERIC = 5                                  # include/sd_b200.h: non-finite result / non-positive pivot
SENTINEL = np.float32(-12345.5)


def _features_like(rng, n, d):
    """HOG-like design matrix: non-negative, bounded by 0.4, correlated columns, bias column of ones."""
    base = rng.random((n, 8)).astype(np.float32)
    mix = rng.random((8, d)).astype(np.float32)
    A = np.clip(0.05 * (base @ mix) + 0.1 * rng.random((n, d)).astype(np.float32), 0, 0.4).astype(np.float32)
    A[:, -1] = 1.0
    return A


def _ulps(a, b):
    return abs(int(np.array([a, b], np.float32).view(np.int32).astype(np.int64) @ np.array([1, -1])))


def _solve(sd, G, M, reg, n_train, pitch, mode=0, lower=np.nan):
    """sd_solve_gram (Cholesky solver, gram mode `mode`) on the upper triangle and right-hand sides of G, laid out with the given
    pitch inside a buffer whose lower triangle and pad columns hold `lower` / NaN and whose guard rows before and after hold
    SENTINEL.  Returns (rc, error, X, lambda, buffer, geometry)."""
    import torch
    from superviseddescent_b200 import _capi
    D = G.shape[0]
    w = D + M
    ldg, shift = CR.pitch(pitch, w)
    g0 = CR.g_offset(ldg, shift)                                # G's first float
    h = np.full(g0 + D * ldg + CR.GUARD_ROWS * ldg, SENTINEL, np.float32)
    body = np.full((D, ldg), np.nan, np.float32)
    body[:, :w] = G[:, :w]
    body[np.tril_indices(D, -1)] = lower
    h[g0:g0 + D * ldg] = body.ravel()
    buf = torch.from_numpy(h).cuda()
    X = torch.full((D, M), float(SENTINEL), dtype=torch.float32, device="cuda")
    lam = C.c_float(0)
    ctx = sd.default_context()
    ctx.set_gram_mode(mode)
    ctx.set_solver("cholesky")
    assert (buf.data_ptr() + 4 * g0) % 16 == 4 * g0 % 16, "the buffer's allocation is not 16-byte aligned"
    try:
        rc = _capi.lib().sd_solve_gram(ctx.h, _capi.ptr(buf.data_ptr() + 4 * g0), C.c_int64(ldg), D, M,
                                       C.byref(_capi.RegulariserC(*reg)), n_train, _capi.ptr(X), C.byref(lam))
        err = _capi.lib().sd_last_error(ctx.h).decode() if rc else ""
        torch.cuda.synchronize()
    finally:
        ctx.set_gram_mode(0)
        ctx.set_solver("cholesky")
    return rc, err, X.cpu().numpy(), lam.value, buf.cpu().numpy(), (g0, ldg, w)


def _untouched(out, geom, D):
    g0, ldg, w = geom
    assert np.array_equal(out[:g0].view(np.uint32), np.full(g0, SENTINEL).view(np.uint32)), "write before G"
    tail = out[g0 + D * ldg:]
    assert np.array_equal(tail.view(np.uint32), np.full(tail.size, SENTINEL).view(np.uint32)), "write after G"
    assert np.all(np.isnan(out[g0:g0 + D * ldg].reshape(D, ldg)[:, w:])), "write into the pad columns"


def _report(name, r):
    worst = CR.worst_by_tile(r)
    print(f"{name}: worst error / bar per (128-row block, 64-column group):")
    for i, row in enumerate(worst):
        print(f"  rows {i * 128:5d}: " + " ".join(f"{v:8.3f}" for v in row))


@pytest.mark.parametrize("case", CR.SWEEP, ids=CR.sweep_id)
def test_solve_gram_vs_float64(sd, case):
    D, M, cond, mode, pitch, typ, last = case
    G, reg = CR.sweep_system(case)
    rc, err, X, lam, out, geom = _solve(sd, G, M, reg, CR.N_DESIGN, pitch, mode)
    routes = CR.case_routes(case)
    print(f"{CR.sweep_id(case)}: tensor-core / SIMT SYRK launches {CR.syrk_launches(routes)}, panels (tensor cores, tail): {routes}")
    _untouched(out, geom, D)
    T = CR.Truth(CR.regularise(G, lam, bool(last)), M)
    if rc == SD_ERR_NUMERIC and mode == 1:
        # one TF32 pass may not factor a system whose smallest eigenvalue its split error can reach; it must say so
        print(f"{CR.sweep_id(case)}: {err} (lambda_min {T.smin():.1e}, split reach {CR.SPLIT_UPDATE[mode] * T.utu_norm():.1e})")
        assert T.split_can_break(mode) and "not positive definite" in err
        return
    assert rc == 0, err
    assert np.all(np.isfinite(X))
    rc0, _, X0, lam0, _, _ = _solve(sd, G, M, reg, CR.N_DESIGN, pitch, mode, lower=0.0)     # the lower triangle is not an input
    assert rc0 == 0 and lam0 == lam
    assert np.array_equal(X.view(np.uint32), X0.view(np.uint32)), "X depends on the lower triangle"
    if D >= 2049:                                               # look-ahead: updates in panel order whatever the timing
        _, _, X1, _, _, _ = _solve(sd, G, M, reg, CR.N_DESIGN, pitch, mode)
        assert np.array_equal(X.view(np.uint32), X1.view(np.uint32)), "the same solve twice differs"
    if typ == 1:
        ref = CR.lambda_matrix_norm(G, reg[1], CR.N_DESIGN)
        assert _ulps(lam, ref) <= 1, (lam, ref)
    else:
        assert lam == np.float32(reg[1])
    eta, eta_ref = T.eta(X[:-1]).max(), T.eta_spotrs().max()
    fwd = np.linalg.norm(X[:-1] - T.w) / np.linalg.norm(T.w)
    if mode == 1:
        print(f"{CR.sweep_id(case)}: eta {eta:.2e} (spotrs {eta_ref:.2e}, allowed excess {T.eta_excess(mode):.2e}), "
              f"forward error {fwd:.2e}")
    else:
        bw = T.bar_w(mode)
        r = CR.ratio(X[:-1], T.w, bw)
        rb = float(np.max(np.abs(X[-1] - T.xb) / T.bar_xb(bw)))
        print(f"{CR.sweep_id(case)}: error / bar {r.max():.4f} (bias row {rb:.4f}), eta {eta:.2e} (spotrs {eta_ref:.2e}), "
              f"forward error {fwd:.2e}")
        if r.max() > 1.0:
            _report(CR.sweep_id(case), r)
        assert r.max() <= 1.0
        assert rb <= 1.0
    assert eta <= eta_ref + T.eta_excess(mode)


# ---- learn path --------------------------------------------------------------------------------------------------------------
def _learn_centred(sd, A, B, reg):
    """sd_centre_features + sd_learn_centred on a device copy of A: (mu, centred A, X, Xc, lambda)"""
    import torch
    from superviseddescent_b200 import _capi
    N, D = A.shape
    M = B.shape[1]
    ctx = sd.default_context()
    ctx.set_solver("cholesky")
    lib = _capi.lib()
    dA, dB = torch.from_numpy(A.copy()).cuda(), torch.from_numpy(B).cuda()
    mu = torch.full((D,), float(SENTINEL), dtype=torch.float32, device="cuda")
    X = torch.full((D, M), float(SENTINEL), dtype=torch.float32, device="cuda")
    Xc = torch.full((D, M), float(SENTINEL), dtype=torch.float32, device="cuda")
    regc = _capi.RegulariserC(*reg)
    assert lib.sd_centre_features(ctx.h, None, _capi.ptr(dA), C.c_int64(D), N, D, N, C.byref(regc), _capi.ptr(mu)) == 0
    lam = C.c_float(0)
    rc = lib.sd_learn_centred(ctx.h, None, _capi.ptr(dA), C.c_int64(D), _capi.ptr(dB), C.c_int64(M), N, D, M, C.byref(regc), N, 0,
                              _capi.ptr(mu), _capi.ptr(X), _capi.ptr(Xc), C.byref(lam))
    assert rc == 0, lib.sd_last_error(ctx.h)
    return mu.cpu().numpy(), dA.cpu().numpy(), X.cpu().numpy(), Xc.cpu().numpy(), lam.value


def _check_learn(sd, A, B, reg, name):
    N, D = A.shape
    mu, Ac, X, Xc, lam = _learn_centred(sd, A, B, reg)
    mu_ref, Ac_ref = CR.centre_restated(A, bool(reg[2]))
    assert np.array_equal(mu.view(np.uint32), mu_ref.view(np.uint32)), "column means"
    assert np.array_equal(Ac.view(np.uint32), Ac_ref.view(np.uint32)), "centred rows"
    lam_true = reg[1] * np.linalg.norm(R.gram_ref(A)) / N
    lbar = CR.lambda_bar(A, Ac, mu, reg[1])
    assert abs(lam - lam_true) <= lbar, (lam, lam_true, lbar)
    T = CR.learn_truth(Ac, B, lam, bool(reg[2]))
    bw = T.bar_w(0)
    r = CR.ratio(Xc[:-1], T.w, bw)
    bxb = T.bar_xb(bw)
    rc_ = float(np.max(np.abs(Xc[-1] - T.xb) / bxb))
    w64 = X[:-1].astype(np.float64)
    shift = mu[:-1].astype(np.float64) @ w64
    x_true = T.xb - mu[:-1].astype(np.float64) @ T.w
    rx = float(np.max(np.abs(X[-1] - x_true) / (bxb + np.abs(mu[:-1].astype(np.float64)) @ bw + 2 * R.U * np.abs(x_true))))
    fwd = np.linalg.norm(Xc[:-1] - T.w) / np.linalg.norm(T.w)
    print(f"{name}: lambda {lam:.7g} (float64 {lam_true:.7g}, bar {lbar:.1e}); error / bar {r.max():.4f}, bias c' {rc_:.4f}, "
          f"bias {rx:.4f}; forward error {fwd:.2e}")
    if r.max() > 1.0:
        _report(name, r)
    assert r.max() <= 1.0 and rc_ <= 1.0 and rx <= 1.0
    assert np.array_equal(X[:-1].view(np.uint32), Xc[:-1].view(np.uint32)), "Xc rows 0..D-2 differ from X"
    # the bias: X_b = (float)(c' - mu.w), Xc_b = (float)c' from the same c' in double
    assert np.all(np.abs(Xc[-1] - (X[-1].astype(np.float64) + shift)) <= R.U * (np.abs(Xc[-1]) + np.abs(X[-1])) + 1e-12 * np.abs(mu[:-1]) @ np.abs(w64))
    # the centred rows with Xc predict what the rows with X predict
    A64, Ac64 = A.astype(np.float64), Ac.astype(np.float64)
    pa, pbar_a = R.predict_ref(A64, X)
    pc, pbar_c = R.predict_ref(Ac64, Xc)
    ebar = pbar_a + pbar_c + R.U * np.abs(Ac64[:, :-1]) @ np.abs(w64) + R.U * (np.abs(X[-1]) + np.abs(Xc[-1]))
    assert np.max(np.abs(pa - pc) / ebar) <= 1.0
    return mu, X, lam


@pytest.mark.parametrize("D", [257, 700, 2049])
@pytest.mark.parametrize("rows", ["fewer", "more"])
def test_learn_centred_vs_float64(sd, D, rows):
    N = D - 100 if rows == "fewer" else 3 * D
    rng = np.random.default_rng(D + N)
    A = _features_like(rng, N, D)
    B = (0.05 * rng.standard_normal((N, 44))).astype(np.float32)
    reg = (1, 1.5, 0)
    mu, X, lam = _check_learn(sd, A, B, reg, f"D={D} N={N}")
    assert mu[:-1].any() and mu[-1] == 0
    lr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False))
    lr.learn(A, B)
    assert np.array_equal(lr.x.cpu().numpy().view(np.uint32), X.view(np.uint32)), "LinearRegressor.learn differs"
    assert lr.last_lambda == lam


@pytest.mark.parametrize("fallback", ["last_column_not_ones", "regularise_last_row"])
def test_learn_centring_fallbacks(sd, fallback):
    """mu = 0 and the rows untouched when the shift would change the problem; the answer still meets its bar"""
    D, N = 700, 2100
    rng = np.random.default_rng(11)
    A = _features_like(rng, N, D)
    last = 0
    if fallback == "last_column_not_ones":
        A[N // 2, -1] = np.float32(1 + 2.0 ** -23)
    else:
        last = 1
    B = (0.05 * rng.standard_normal((N, 44))).astype(np.float32)
    mu, X, lam = _check_learn(sd, A, B, (1, 1.5, last), fallback)
    assert not mu.any()


# ---- small LU ----------------------------------------------------------------------------------------------------------------
def _lu_system(D, M, seed):
    rng = np.random.default_rng(seed)
    G = np.zeros((D, D + M), np.float32)
    S = rng.standard_normal((D, D)).astype(np.float32)
    G[:, :D] = np.triu(S + S.T)
    G[np.arange(D), np.arange(D)] += np.float32(0.5 * D)
    G[:, D:] = rng.standard_normal((D, M)).astype(np.float32)
    if D >= 3:
        # column 0 (the mirror of row 0): |t| = |-t| is its largest entry, in rows 1 and D - 1 -- different warps of the
        # pivot search for D >= 33, so the cross-warp tie-break decides; the first (row 1) must win
        t = np.float32(4 * D + 64)
        G[0, 0], G[0, 1], G[0, D - 1] = 0.25, t, -t
        col = np.abs(G[0, :D])
        assert col.max() == t and np.count_nonzero(col == t) == 2
    return G


@pytest.mark.parametrize("D", [1, 2, 31, 32, 33, 128, 255, 256])
def test_small_lu_bit_for_bit(sd, D):
    for M in (1, 7, 136):
        G = _lu_system(D, M, D * 100 + M)
        reg = (0, 0.5, 0)
        rc, err, X, lam, out, geom = _solve(sd, G, M, reg, 1, "tight")
        assert rc == 0, err
        _untouched(out, geom, D)
        Xr, singular = CR.lu_restated(CR.regularise(G, lam, False), M)
        assert not singular
        assert np.array_equal(X.view(np.uint32), Xr.view(np.uint32)), f"D={D} M={M}"


def test_small_lu_matrix_norm_and_singular(sd):
    D, M = 200, 7
    G = _lu_system(D, M, 5)
    rc, err, X, lam, _, _ = _solve(sd, G, M, (1, 0.01, 1), 77, "odd")
    assert rc == 0, err
    ref = CR.lambda_matrix_norm(G, 0.01, 77)
    assert _ulps(lam, ref) <= 1, (lam, ref)
    Xr, _ = CR.lu_restated(CR.regularise(G, lam, True), M)
    assert np.array_equal(X.view(np.uint32), Xr.view(np.uint32))
    # exactly singular: a rank-one matrix of powers of two leaves an exact zero pivot after the first step
    v = np.array([1, 2, 4, 8, 16], np.float32)
    Gs = np.hstack([np.triu(np.outer(v, v)), np.ones((5, 2), np.float32)]).astype(np.float32)
    assert CR.lu_restated(Gs, 2)[1]
    rc, err, _, _, _, _ = _solve(sd, Gs, 2, (0, 0.0, 1), 1, "tight")
    print("singular:", rc, err)
    assert rc == SD_ERR_NUMERIC and "singular" in err

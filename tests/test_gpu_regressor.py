"""GPU parity of LinearRegressor / SupervisedDescentOptimiser (C ABI) against the reference's literals
and the CPU oracle."""
import numpy as np
import pytest

import known_answers as K
from conftest import rel_err
from test_oracle import run_lr_cases, run_sdo_cases

pytestmark = pytest.mark.gpu
TOL = 1e-4


class GpuBackend:
    def __init__(self, sd):
        self.sd = sd

    def learn(self, data, labels, reg):
        lr = self.sd.LinearRegressor(self.sd.Regulariser(self.sd.RegularisationType(reg[0]), reg[1], reg[2]))
        assert lr.learn(np.asarray(data, np.float32), np.asarray(labels, np.float32)) is True   # regressors.hpp:349
        return lr.x.cpu().numpy()

    def _lr(self, X):
        import torch
        lr = self.sd.LinearRegressor()
        lr._ctx()
        lr.x = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).cuda()
        return lr

    def predict(self, values, X):
        return self._lr(X).predict(np.asarray(values, np.float32)).cpu().numpy()

    def residual(self, data, labels, X):
        return self._lr(X).test(np.asarray(data, np.float32), np.asarray(labels, np.float32))

    def train(self, x_gt, x0, y, h, n_reg, callback=None):
        sdo = self.sd.SupervisedDescentOptimiser([self.sd.LinearRegressor() for _ in range(n_reg)])
        cb = (lambda cur: callback(cur.cpu().numpy())) if callback else None
        xf = sdo.train(x_gt, x0, y, h, cb)
        return sdo, xf.cpu().numpy()

    def test(self, sdo, x0, y, h):
        return sdo.test(x0, y, h).cpu().numpy()


def test_linear_regressor_reference_literals(sd):
    rep = run_lr_cases(GpuBackend(sd))
    print("gpu", [(n, f"{e:.2e}") for n, e in rep])


def test_optimiser_reference_literals(sd):
    rep = run_sdo_cases(GpuBackend(sd))
    print("gpu", [(r[0], f"{r[1]:.2e}", f"{r[2]:.2e}") for r in rep])


def _features_like(rng, n, d):
    """HOG-like design matrix: non-negative, bounded by 0.4, correlated columns, bias column of ones."""
    base = rng.random((n, 8)).astype(np.float32)
    mix = rng.random((8, d)).astype(np.float32)
    A = np.clip(0.05 * (base @ mix) + 0.1 * rng.random((n, d)).astype(np.float32), 0, 0.4).astype(np.float32)
    A[:, -1] = 1.0
    return A


@pytest.mark.parametrize("mode", [2, 0, 3, 1])
def test_gram_and_solve_vs_oracle(sd, oracle, mode):
    """[AtA | Atb] and the regularised solve at a size that takes the tensor-core SYRK and the blocked
    Cholesky.  mode 2 = fp32 SIMT, 0 = 3xTF32 wgmma (truncated hi), 3 = unbiased 3xTF32, 1 = single-pass TF32 (looser)."""
    import ctypes as C
    import torch
    from superviseddescent_b200 import _capi
    rng = np.random.default_rng(123)
    n, d, m = 1500, 700, 44
    A = _features_like(rng, n, d)
    B = (0.05 * rng.standard_normal((n, m))).astype(np.float32)
    ctx = sd.default_context()
    ctx.set_gram_mode(mode)
    try:
        dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
        ldg = d + m
        G = torch.zeros((d, ldg), dtype=torch.float32, device="cuda")
        rc = _capi.lib().sd_gram(ctx.h, _capi.ptr(dA), C.c_int64(d), _capi.ptr(dB), C.c_int64(m), n, d, m, _capi.ptr(G), C.c_int64(ldg))
        assert rc == 0, _capi.lib().sd_last_error(ctx.h)
        Gh = G.cpu().numpy()
        A64 = A.astype(np.float64)
        Gd = A64.T @ A64
        Rd = A64.T @ B.astype(np.float64)
        iu = np.triu_indices(d)
        e_g = np.max(np.abs(Gh[:, :d][iu] - Gd[iu])) / np.max(np.abs(Gd))
        e_r = rel_err(Gh[:, d:], Rd)
        print(f"mode {mode}: gram rel err {e_g:.2e}, Atb rel err {e_r:.2e}")
        tol = 2e-3 if mode == 1 else 2e-6
        assert e_g <= tol and e_r <= tol * 5
        reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)
        lr = sd.LinearRegressor(reg)
        lr.learn(dA, dB)
        X = lr.x.cpu().numpy()
        Xo, lam = oracle.solve(A, B, oracle.Regulariser(1, 1.5, 0), 1)      # float64 truth
        Xf, lamf = oracle.solve(A, B, oracle.Regulariser(1, 1.5, 0), 0)     # float32 restatement (Eigen-like)
        print(f"mode {mode}: lambda gpu {lr.last_lambda:.6g} oracle {lam:.6g}; X rel err vs f64 {rel_err(X, Xo):.2e}; f32 oracle vs f64 {rel_err(Xf, Xo):.2e}")
        assert abs(lr.last_lambda - lam) <= 1e-5 * lam * (100 if mode == 1 else 1)
        assert rel_err(X, Xo) <= (5e-2 if mode == 1 else TOL)
        pred = lr.predict(dA[:64]).cpu().numpy()
        assert rel_err(pred, oracle.predict(A[:64], X)) <= TOL
        print("timings", ctx.solver_timings())
    finally:
        ctx.set_gram_mode(0)


def test_small_lu_path_is_bit_faithful_to_the_oracle_solver(sd, oracle):
    """D <= 256 uses the partial-pivot LU that restates the oracle's operation order."""
    rng = np.random.default_rng(9)
    A = rng.standard_normal((300, 20)).astype(np.float32)
    B = rng.standard_normal((300, 6)).astype(np.float32)
    for reg in [(0, 0.0, True), (1, 2.0, True), (1, 0.5, False)]:
        lr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType(reg[0]), reg[1], reg[2]))
        lr.learn(A, B)
        Xo, lam = oracle.solve(A, B, oracle.Regulariser(reg[0], reg[1], int(reg[2])), 0)
        assert rel_err(lr.x.cpu().numpy(), Xo) <= 1e-5
        assert abs(lr.last_lambda - lam) <= 1e-6 * max(lam, 1e-6)


def test_singular_system_is_reported(sd):
    with pytest.raises(RuntimeError):
        sd.LinearRegressor().learn(np.zeros((1, 1), np.float32), np.ones((1, 1), np.float32))   # test_LinearRegressor1D.cpp:29-38


def test_cascade_with_ied_normalisation_vs_oracle(sd, oracle, golden):
    """train() with InterEyeDistanceNormalisation and a host projection functor, against the oracle cascade."""
    rng = np.random.default_rng(17)
    L, n = 6, 80
    ids = [str(i) for i in range(L)]
    x_gt = (rng.random((n, 2 * L)) * 50 + 20).astype(np.float32)
    x0 = (x_gt + rng.standard_normal((n, 2 * L)) * 3).astype(np.float32)
    W = rng.standard_normal((2 * L, 9)).astype(np.float32) * 0.01

    def h(row, level, idx):
        f = np.tanh(row @ W)
        return np.concatenate([f, [1.0]]).astype(np.float32)

    regs = [sd.Regulariser(sd.RegularisationType.MatrixNorm, 0.5, False) for _ in range(3)]
    norm = sd.InterEyeDistanceNormalisation(ids, ["0", "1"], ["4"])
    sdo = sd.SupervisedDescentOptimiser([sd.LinearRegressor(r) for r in regs], norm)
    xf = sdo.train(x_gt, x0, None, h).cpu().numpy()
    oregs = [oracle.Regulariser(1, 0.5, 0) for _ in range(3)]
    w, xo, rc = oracle.cascade_train(x_gt, x0, None, oregs, [10] * 3, h, norm=([0, 1], [4]), precision=0)
    assert rel_err(xf, xo) <= TOL
    for k in range(3):
        assert rel_err(sdo.regressors[k].x.cpu().numpy(), w[k]) <= 2e-3     # ill-conditioned toy system: weights looser than outputs
    xt = sdo.test(x0[:10], None, h).cpu().numpy()
    assert rel_err(xt, oracle.cascade_apply(x0[:10], None, w, h, norm=([0, 1], [4]))) <= TOL


def test_pose_estimation_example_config2(sd, oracle):
    """BASELINE config 2 (examples/pose_estimation.cpp) on the GPU: host projection functor, GPU learn/predict,
    against the oracle cascade on the same seeded training set."""
    import pose_example as P
    x_tr, y_tr, x0 = P.training_set()
    regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 2.0, True)) for _ in range(3)]
    sdo = sd.SupervisedDescentOptimiser(regs)
    res = []
    xf = sdo.train(x_tr, x0, y_tr, P.projection, lambda cur: res.append(K.nlsr(cur.cpu().numpy(), x_tr))).cpu().numpy()
    oregs = [oracle.Regulariser(1, 2.0, 1) for _ in range(3)]
    w, xo, rc = oracle.cascade_train(x_tr, x0, y_tr, oregs, [20] * 3, P.projection, None, 0)
    print("gpu pose residuals", res, "final x rel err vs oracle", rel_err(xf, xo))
    assert rel_err(xf, xo) <= 1e-4
    for k in range(3):
        assert rel_err(sdo.regressors[k].x.cpu().numpy(), w[k]) <= 1e-3
    pred = sdo.predict(P.TEST_INIT, P.TEST_LANDMARKS, P.projection).cpu().numpy()[0]
    ref = oracle.cascade_apply(P.TEST_INIT, P.TEST_LANDMARKS, w, P.projection, None)[0]
    print("predicted pitch/yaw/roll", pred[:3], "oracle", ref[:3])
    assert np.max(np.abs(pred - ref)) <= 1e-4 * np.max(np.abs(ref))
    assert np.all(np.abs(pred[:3] - np.array([11.0, -25.0, -10.0])) < 6.0)


@pytest.mark.parametrize("D,M,pad", [(257, 1, 0), (300, 8, 0), (384, 44, 0), (385, 44, 1), (513, 3, 2), (640, 70, 0),
                                     (1000, 44, 3), (1153, 136, 0), (2600, 44, 0), (4097, 136, 0), (2600, 44, 1)])
def test_blocked_cholesky_shapes(sd, D, M, pad):
    """sd_solve_gram on well-conditioned SPD systems of awkward shapes: D just above the LU limit, odd numbers of
    128-blocks (a panel with a single block), ragged last blocks, right-hand sides wider than one column tile, and
    leading dimensions that are not a multiple of 4 (scalar staging, SIMT trailing updates instead of TMA), and early panels
    whose tail updates have more tiles than the GPU has SMs (tensor cores, and SIMT on a large matrix at an odd pitch).  Manual
    regularisation lambda = 0.5 is added to the diagonal as regressors.hpp:126-148 does (bias row unregularised)."""
    import ctypes as C
    import torch
    from superviseddescent_b200 import _capi
    rng = np.random.default_rng(D * 7 + M)
    Q = rng.standard_normal((D + 40, D))
    G64 = Q.T @ Q / (D + 40) + np.eye(D)                      # condition number of a few units
    R64 = rng.standard_normal((D, M))
    ldg = D + M + pad
    Gh = np.zeros((D, ldg), np.float32)
    Gh[:, :D] = np.triu(G64)                                  # only the upper triangle is an input
    Gh[:, D:D + M] = R64
    lam = 0.5
    Greg = G64.copy()
    Greg[np.arange(D - 1), np.arange(D - 1)] += np.float32(lam)   # regularise_last_row = false
    Xo = np.linalg.solve(Greg.astype(np.float32).astype(np.float64), R64.astype(np.float32).astype(np.float64))
    ctx = sd.default_context()
    G = torch.from_numpy(Gh).cuda()
    X = torch.zeros((D, M), dtype=torch.float32, device="cuda")
    reg = _capi.RegulariserC(0, lam, 0)
    lam_out = C.c_float(0)
    rc = _capi.lib().sd_solve_gram(ctx.h, _capi.ptr(G), C.c_int64(ldg), D, M, C.byref(reg), 1, _capi.ptr(X), C.byref(lam_out))
    assert rc == 0, _capi.lib().sd_last_error(ctx.h)
    assert abs(lam_out.value - lam) < 1e-7
    err = rel_err(X.cpu().numpy(), Xo)
    print(f"D={D} M={M} ldg={ldg}: X rel err {err:.2e}")
    assert err <= 2e-5


def test_colpiv_qr_solver_rank_diagnostic(sd, capsys):
    """ColPivHouseholderQRSolver (regressors.hpp:245-306): same solution as the LU solver on regular systems; the numerical rank
    of the regularised AtA (the diagnostic that solver exists for, :288-293) comes from a diagonally pivoted Cholesky."""
    rng = np.random.default_rng(3)
    n, d, m = 600, 300, 5
    A = rng.random((n, d)).astype(np.float32)
    A[:, -1] = 1.0
    B = rng.standard_normal((n, m)).astype(np.float32)
    lu = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 0.5, True))
    qr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 0.5, True), solver=sd.ColPivHouseholderQRSolver())
    lu.learn(A, B)
    qr.learn(A, B)
    assert qr.last_rank == d
    assert np.array_equal(qr.x.cpu().numpy(), lu.x.cpu().numpy())
    # rank-deficient: 40 duplicated columns, lambda = 0
    A2 = A.copy()
    A2[:, 10:50] = A2[:, 100:140]
    q0 = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 0.0, True), solver=sd.ColPivHouseholderQRSolver())
    assert q0.learn(A2, B) is True                      # learn() always returns true (regressors.hpp:349)
    assert q0.last_rank == d - 40
    assert f"(The rank is {d - 40}, full rank would be {d}). Increase lambda." in capsys.readouterr().out
    # ... and regular again once lambda > 0
    q1 = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 1.0, True), solver=sd.ColPivHouseholderQRSolver())
    q1.learn(A2, B)
    assert q1.last_rank == d and np.isfinite(q1.x.cpu().numpy()).all()
    # small systems (the LU route, D <= 256) report their rank too
    A3 = rng.random((50, 6)).astype(np.float32)
    A3[:, 5] = A3[:, 0] + A3[:, 1]
    q2 = sd.LinearRegressor(sd.Regulariser(), solver=sd.ColPivHouseholderQRSolver())
    q2.learn(A3, rng.standard_normal((50, 2)).astype(np.float32))
    assert q2.last_rank == 5


def test_conjugate_gradient_route_matches_the_factorisation(sd):
    """sd_set_solver(1): CG on the tensor cores for the centred, MatrixNorm-regularised system (well conditioned) must give the
    weights of the blocked Cholesky; an ill-conditioned system (tiny manual lambda) must fall back to the factorisation and say so
    (a negative iteration count)."""
    ctx = sd.default_context()
    A = _features_like(np.random.default_rng(31), 2500, 1800)
    B = (0.05 * np.random.default_rng(32).standard_normal((2500, 44))).astype(np.float32)
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)
    chol = sd.LinearRegressor(reg)
    chol.learn(A, B)
    assert ctx.solver_iterations() == 0
    ctx.set_solver("cg")
    try:
        cg = sd.LinearRegressor(reg)
        cg.learn(A, B)
        its = ctx.solver_iterations()
        e = rel_err(cg.x.cpu().numpy(), chol.x.cpu().numpy())
        A64 = A.astype(np.float64)
        G = A64.T @ A64
        lam = 1.5 * np.linalg.norm(G) / A.shape[0]
        R = np.eye(G.shape[0]) * lam
        R[-1, -1] = 0
        Xt = np.linalg.solve(G + R, A64.T @ B.astype(np.float64))
        print(f"CG: {its} iterations; weights vs Cholesky {e:.2e}; vs float64 CG {rel_err(cg.x.cpu().numpy(), Xt):.2e} / Cholesky {rel_err(chol.x.cpu().numpy(), Xt):.2e}; {ctx.solver_timings()}")
        assert 3 <= its <= 200
        assert e <= 2e-5
        assert rel_err(cg.x.cpu().numpy(), Xt) <= 1e-4
        # 136 right-hand sides (68 landmarks): two tile rows of the product
        B2 = (0.05 * np.random.default_rng(33).standard_normal((2500, 136))).astype(np.float32)
        cg2 = sd.LinearRegressor(reg)
        cg2.learn(A, B2)
        assert ctx.solver_iterations() >= 3
        ctx.set_solver("cholesky")
        ch2 = sd.LinearRegressor(reg)
        ch2.learn(A, B2)
        assert rel_err(cg2.x.cpu().numpy(), ch2.x.cpu().numpy()) <= 2e-5
        # tiny lambda: condition number ~1e6, CG stalls -> the factorisation answers
        ctx.set_solver("cg")
        hard = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 1e-4, True))
        hard.learn(A, B)
        its_hard = ctx.solver_iterations()
        ctx.set_solver("cholesky")
        ref = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 1e-4, True))
        ref.learn(A, B)
        print(f"tiny lambda: CG gave up after {-its_hard} iterations")
        assert its_hard < 0                                 # CG ran, gave up, and the factorisation answered
        assert ctx.solver_iterations() == 0
        assert np.array_equal(hard.x.cpu().numpy(), ref.x.cpu().numpy())
        assert np.isfinite(hard.x.cpu().numpy()).all()
        pa, pb = A @ hard.x.cpu().numpy(), A @ ref.x.cpu().numpy()
        assert rel_err(pa, pb) <= 1e-3
    finally:
        ctx.set_solver("cholesky")


# (D - 1, M): right-hand sides up to 64 take the narrow (64-column) product, more take 128-column tiles, 192 is the CG cap;
# D - 1 = 1799 and 3000 leave a padded, partial last strip of the strip-major operand, 2048 fills it exactly
@pytest.mark.parametrize("n,m", [(1799, 1), (1799, 44), (1799, 64), (1799, 65), (1799, 136), (1799, 192), (1799, 193),
                                 (2048, 44), (3000, 44), (3000, 136)])
def test_conjugate_gradient_shapes_match_float64_and_the_factorisation(sd, n, m):
    """sd_set_solver(1): CG on the tensor cores for the centred, MatrixNorm-regularised system (well conditioned) must converge
    (a positive iteration count) to the weights of the blocked Cholesky and of float64; more than 192 right-hand sides are the
    factorisation's job (0: CG not tried)."""
    ctx = sd.default_context()
    d = n + 1
    samples = d + 700
    A = _features_like(np.random.default_rng(31 + n), samples, d)
    B = (0.05 * np.random.default_rng(32 + m).standard_normal((samples, m))).astype(np.float32)
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)
    chol = sd.LinearRegressor(reg)
    chol.learn(A, B)
    assert ctx.solver_iterations() == 0
    ctx.set_solver("cg")
    try:
        cg = sd.LinearRegressor(reg)
        cg.learn(A, B)
        its = ctx.solver_iterations()
    finally:
        ctx.set_solver("cholesky")
    A64 = A.astype(np.float64)
    G = A64.T @ A64
    lam = 1.5 * np.linalg.norm(G) / samples
    Rg = np.eye(d) * lam
    Rg[-1, -1] = 0
    Xt = np.linalg.solve(G + Rg, A64.T @ B.astype(np.float64))
    Xcg, Xch = cg.x.cpu().numpy(), chol.x.cpu().numpy()
    e = rel_err(Xcg, Xch)
    print(f"D={d} M={m}: CG {its} iterations; weights vs Cholesky {e:.2e}; vs float64 CG {rel_err(Xcg, Xt):.2e} / Cholesky {rel_err(Xch, Xt):.2e}")
    if m > 192:
        assert its == 0
        assert np.array_equal(Xcg, Xch)
        return
    assert 3 <= its <= 200
    assert e <= 2e-5
    assert rel_err(Xcg, Xt) <= 1e-4

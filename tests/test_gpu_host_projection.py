"""Cascade levels on the caller's host projection (sd_train_level_host_projected, sd_apply_level_host_projected, and the Python
mirror's HostProjection / RowwiseProjection).

A host callback that writes the rows a device callback writes must give the device-projection level bit for bit, for any
staging-half size, and be called batch by batch in ascending order; the pose example through RowwiseProjection must give the
plain-functor route bit for bit; a large random-feature projection must train in chunks within the bars of
test_gpu_projection.py and reproducibly; errors and bad descriptors are refused as for the device callback."""
import ctypes as C
import gc

import numpy as np
import pytest

import pose_example as PE
from conftest import rel_err

pytestmark = pytest.mark.gpu


def _random_data(n, P, seed=9):
    rng = np.random.default_rng(seed)
    x_gt = rng.uniform(-1, 1, (n, P)).astype(np.float32)
    x0 = (x_gt + rng.normal(0, 0.3, (n, P))).astype(np.float32)
    return x_gt, x0


def _features(x, features=3000, seed=5):
    """cos(x W + b) with a last column of ones: n x (features + 1) float32, each row independent of the others"""
    rng = np.random.default_rng(seed)
    W = rng.standard_normal((x.shape[1], features)).astype(np.float32)
    b = rng.uniform(0, 2 * np.pi, features).astype(np.float32)
    acc = np.broadcast_to(b, (x.shape[0], features)).copy()
    for p in range(x.shape[1]):
        acc += x[:, p:p + 1] * W[p]
    return np.concatenate([np.cos(acc), np.ones((x.shape[0], 1), np.float32)], axis=1).astype(np.float32)


def _optimiser(sd, levels, solver=None):
    return sd.SupervisedDescentOptimiser([sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), None, solver)
                                          for _ in range(levels)])


def _batches(n, chunk, per_half, passes):
    """the (first_row, rows) calls of the host callback: per chunk, batches of at most per_half rows; passes: "train" (every
    chunk, then every chunk but the last again) or "apply" (every chunk)"""
    chunks = [(r0, min(chunk, n - r0)) for r0 in range(0, n, chunk)]
    if passes == "train":
        chunks = chunks + chunks[:-1]
    return [(r0 + b, min(per_half, rows - b)) for r0, rows in chunks for b in range(0, rows, per_half)]


# ---- bit identity with the device callback ----------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [3000, 1100])
@pytest.mark.parametrize("half", ["default", "one row", "three rows"])
def test_host_callback_is_the_device_callback(sd, chunk, half):
    import torch
    ctx = sd.default_context()
    lib, ptr = sd._capi.lib(), sd._capi.ptr
    n, P = 3000, 10
    x_gt, x0 = _random_data(n, P)
    F = _features(x0)
    D = F.shape[1]
    ld_out = (D + 3) // 4 * 4
    stage = {"default": 0, "one row": 4 * ld_out, "three rows": 3 * 4 * ld_out + 12}[half]
    per_half = {"default": (48 << 20) // (4 * ld_out), "one row": 1, "three rows": 3}[half]
    Fd = torch.from_numpy(F).cuda()
    cur, gt = torch.from_numpy(x0).cuda(), torch.from_numpy(x_gt).cuda()
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()

    def on_device(user, c, lvl, d_x, ldx, first_row, rows, d_out, ld):
        return lib.sd_memcpy2d_d2d(C.c_void_p(c), C.c_void_p(d_out), C.c_size_t(4 * ld), C.c_void_p(Fd.data_ptr() + 4 * D * first_row),
                                   C.c_size_t(4 * D), C.c_size_t(4 * D), C.c_size_t(rows))
    dev_fn = sd._capi.ProjectFn(on_device)
    dev = sd._capi.LevelProjectionC(dev_fn, None, 0, D)
    calls, inputs = [], []

    def on_host(user, lvl, h_x, ldx, first_row, rows, h_out, ld):
        calls.append((first_row, rows))
        x = np.ctypeslib.as_array((C.c_float * (rows * ldx)).from_address(h_x)).reshape(rows, ldx)
        inputs.append(ldx == P and ld == ld_out and np.array_equal(x, x0[first_row:first_row + rows]))   # checked after the call
        out = np.ctypeslib.as_array((C.c_float * (rows * ld)).from_address(h_out)).reshape(rows, ld)
        out[:, :D] = F[first_row:first_row + rows]
        out[:, D:] = np.nan                                          # padding of the staged rows is never uploaded
        return 0
    host_fn = sd._capi.HostProjectFn(on_host)
    host = sd._capi.LevelHostProjectionC(host_fn, None, 0, D, stage)
    ld, lda = (D + P + 3) // 4 * 4, (D + 3) // 4 * 4
    outs = []
    for hosted in (False, True):
        buf = torch.full((chunk, ld), 7.0, device="cuda")
        X, nxt, lam = torch.empty((D, P), device="cuda"), torch.empty_like(cur), C.c_float(0)
        train = lib.sd_train_level_host_projected if hosted else lib.sd_train_level_projected
        rc = train(ctx.h, None, C.byref(host if hosted else dev), ptr(cur), ptr(gt), n, P, n, None, None, 0, C.byref(reg), 0, ptr(buf), ld,
                   chunk, ptr(X), ptr(nxt), C.byref(lam))
        assert rc == 0, lib.sd_last_error(ctx.h).decode()
        abuf = torch.empty((chunk, lda), device="cuda")
        applied = torch.empty_like(cur)
        apply = lib.sd_apply_level_host_projected if hosted else lib.sd_apply_level_projected
        rc = apply(ctx.h, C.byref(host if hosted else dev), ptr(cur), n, P, None, None, 0, ptr(X), ptr(abuf), lda, chunk, ptr(applied))
        assert rc == 0, lib.sd_last_error(ctx.h).decode()
        ctx.sync()
        outs.append((X.cpu().numpy(), lam.value, nxt.cpu().numpy(), applied.cpu().numpy()))
    (X0, lam0, nxt0, app0), (X1, lam1, nxt1, app1) = outs
    assert np.array_equal(X0, X1) and lam0 == lam1 and np.array_equal(nxt0, nxt1) and np.array_equal(app0, app1)
    assert calls == _batches(n, chunk, per_half, "train") + _batches(n, chunk, per_half, "apply") and all(inputs)


# ---- the pose example through RowwiseProjection ------------------------------------------------------------------------------
def test_pose_example_rowwise_is_the_plain_functor(sd):
    x_tr, y_tr, x0 = PE.training_set()

    def optimiser():
        return sd.SupervisedDescentOptimiser([sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 2.0, True)) for _ in range(3)])
    plain, piped = optimiser(), optimiser()
    proj = sd.RowwiseProjection(PE.projection, 20)
    seen_plain, seen_piped = [], []
    xp = plain.train(x_tr, x0, y_tr, PE.projection, lambda x: seen_plain.append(x.cpu().numpy())).cpu().numpy()
    xh = piped.train(x_tr, x0, y_tr, proj, lambda x: seen_piped.append(x.cpu().numpy())).cpu().numpy()
    assert piped.chunk_rows == [x_tr.shape[0]] * 3                  # templates: one chunk
    for a, b in zip(plain.regressors, piped.regressors):
        assert np.array_equal(a.x.cpu().numpy(), b.x.cpu().numpy()) and a.last_lambda == b.last_lambda
    assert np.array_equal(xp, xh) and all(np.array_equal(a, b) for a, b in zip(seen_plain, seen_piped))
    tp = plain.test(PE.TEST_INIT, PE.TEST_LANDMARKS, PE.projection).cpu().numpy()
    th = piped.test(PE.TEST_INIT, PE.TEST_LANDMARKS, proj).cpu().numpy()
    print("pose through RowwiseProjection: pitch/yaw/roll", th[0, :3])
    assert np.array_equal(tp, th)
    assert np.array_equal(piped.predict(PE.TEST_INIT, PE.TEST_LANDMARKS, proj).cpu().numpy(), th)


# ---- large D in chunks, the rank diagnostic, reproducibility -----------------------------------------------------------------
class RandomFeatures:
    """_features as a duck-typed HostProjection, one projection per level"""

    def __init__(self, levels):
        self.levels = levels
        self.calls = 0

    def feature_length(self, level):
        return 3001

    def project_host(self, x, level, first_row, out):
        self.calls += 1
        out[:] = _features(x, seed=5 + level)


class FromTable:
    """precomputed rows, as a HostProjection and as a DeviceProjection"""

    def __init__(self, F, on_device):
        import torch
        self.F = torch.from_numpy(F).cuda() if on_device else F
        setattr(self, "project" if on_device else "project_host", self._rows)

    def feature_length(self, level):
        return self.F.shape[1]

    def _rows(self, x, level, first_row, out):
        out[:] = self.F[first_row:first_row + x.shape[0]]


def test_large_random_features_in_chunks(sd):
    n, P = 6000, 10
    x_gt, x0 = _random_data(n, P)
    proj = RandomFeatures(2)
    runs = {}
    for rows in (None, 1700, 1700):
        sdo = _optimiser(sd, 2)
        xf = sdo.train(x_gt, x0, None, proj, rows_per_chunk=rows).cpu().numpy()
        assert sdo.chunk_rows == [rows or n] * 2
        runs.setdefault(rows, []).append(([r.x.cpu().numpy() for r in sdo.regressors], xf, sdo))
    (W1, x1, one), = runs[None]
    (Wa, xa, _), (Wb, xb, _) = runs[1700]
    assert all(np.array_equal(a, b) for a, b in zip(Wa, Wb)) and np.array_equal(xa, xb)      # reproducible for a fixed chunking
    e_w, e_x = max(rel_err(a, b) for a, b in zip(Wa, W1)), rel_err(xa, x1)
    print(f"host projection, D = 3001, 4 chunks vs one: weights {e_w:.2e}, x {e_x:.2e}")
    assert e_w <= 2e-5 and e_x <= 1e-4
    t1 = one.test(x0, None, proj).cpu().numpy()
    tc = one.test(x0, None, proj, rows_per_chunk=1700).cpu().numpy()
    assert rel_err(tc, t1) <= 1e-5


def test_rank_diagnostic_and_device_route_on_the_same_rows(sd):
    n, P = 4000, 10
    x_gt, x0 = _random_data(n, P)
    F = _features(x0)
    results = []
    for on_device in (True, False, False):
        qr = _optimiser(sd, 1, solver=sd.ColPivHouseholderQRSolver())
        xf = qr.train(x_gt, x0, None, FromTable(F, on_device), rows_per_chunk=1500).cpu().numpy()
        results.append((qr.regressors[0].last_rank, qr.regressors[0].x.cpu().numpy(), xf))
    print("ranks, device route and twice the host route:", [r for r, _, _ in results])
    assert results[0][0] == results[1][0] == results[2][0] == 3001
    for rank, X, xf in results[1:]:
        assert np.array_equal(X, results[0][1]) and np.array_equal(xf, results[0][2])


# ---- memory --------------------------------------------------------------------------------------------------------------------
def test_each_level_frees_its_chunk_buffer(sd):
    """The chunk query of a level must see the previous level's buffer freed, by reference counting alone: the level's callback
    holds no reference cycle."""
    import torch
    n, P = 2000, 10
    x_gt, x0 = _random_data(n, P)
    F = _features(x0, features=500)
    chunk_bytes = n * ((F.shape[1] + P + 3) // 4 * 4) * 4
    allocated = []
    sdo = _optimiser(sd, 3)
    query = sdo._chunk_rows

    def checked(*args):
        allocated.append(torch.cuda.memory_allocated())
        return query(*args)
    sdo._chunk_rows = checked
    gc.disable()
    try:
        for run in ("train", "test"):
            allocated.clear()
            if run == "train":
                sdo.train(x_gt, x0, None, FromTable(F, False))
            else:
                sdo.test(x0, None, FromTable(F, False))
            # the level's chunk buffer (chunk_bytes) is gone before the next level's query: at most the small outputs remain
            assert len(allocated) == 3 and max(allocated) - allocated[0] < chunk_bytes // 4, (run, allocated)
    finally:
        gc.enable()


# ---- errors --------------------------------------------------------------------------------------------------------------------
def test_callback_errors_fail_the_level(sd):
    import torch
    ctx = sd.default_context()
    lib, ptr = sd._capi.lib(), sd._capi.ptr
    n, P, D = 64, 6, 9
    x_gt, x0 = _random_data(n, P)
    cur, gt = torch.from_numpy(x0).cuda(), torch.from_numpy(x_gt).cuda()
    ld = (D + P + 3) // 4 * 4
    buf = torch.empty((n, ld), device="cuda")
    X, nxt = torch.empty((D, P), device="cuda"), torch.empty_like(cur)
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    fails = sd._capi.LevelHostProjectionC(sd._capi.HostProjectFn(lambda *a: 3), None, 0, D, 0)
    assert lib.sd_train_level_host_projected(ctx.h, None, C.byref(fails), ptr(cur), ptr(gt), n, P, n, None, None, 0, C.byref(reg), 0,
                                             ptr(buf), ld, n, ptr(X), ptr(nxt), None) == 1
    assert "projection callback returned 3" in lib.sd_last_error(ctx.h).decode()
    assert lib.sd_apply_level_host_projected(ctx.h, C.byref(fails), ptr(cur), n, P, None, None, 0, ptr(X), ptr(buf), ld, n, ptr(nxt)) == 1
    assert "projection callback returned 3" in lib.sd_last_error(ctx.h).decode()

    class Broken(sd.HostProjection):
        def feature_length(self, level):
            return D

        def project_host(self, x, level, first_row, out):
            raise ValueError(f"no features for rows from {first_row}")
    with pytest.raises(ValueError, match="no features for rows from 0"):
        _optimiser(sd, 2).train(x_gt, x0, None, Broken())

    class SecondChunk(Broken):
        def project_host(self, x, level, first_row, out):
            if first_row:
                super().project_host(x, level, first_row, out)
            out[:] = 1.0
    sdo = _optimiser(sd, 1)
    sdo.train(x_gt, x0, None, FromTable(_features(x0, features=D - 1), False))
    with pytest.raises(ValueError, match="no features for rows from 32"):
        sdo.test(x0, None, SecondChunk(), rows_per_chunk=32)
    with pytest.raises(ValueError, match="h returned 3 values for row 0"):
        sdo.test(x0, None, sd.RowwiseProjection(lambda r, level, i: np.zeros(3, np.float32), D))


def test_bad_host_projections_are_refused_before_any_work(sd):
    import torch
    ctx = sd.default_context()
    lib, ptr = sd._capi.lib(), sd._capi.ptr
    n, P, D = 64, 6, 9
    x_gt, x0 = _random_data(n, P)
    cur, gt = torch.from_numpy(x0).cuda(), torch.from_numpy(x_gt).cuda()
    ld = (D + P + 3) // 4 * 4
    buf = torch.empty((n, ld), device="cuda")
    X, nxt = torch.full((D, P), 7.0, device="cuda"), torch.full((n, P), 7.0, device="cuda")
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    calls = []
    F = np.random.default_rng(1).random((n, D)).astype(np.float32)

    def rows(user, level, h_x, ldx, first_row, count, h_out, ld_out):
        calls.append(first_row)
        out = np.ctypeslib.as_array((C.c_float * (count * ld_out)).from_address(h_out)).reshape(count, ld_out)
        out[:, :D] = F[first_row:first_row + count]
        return 0
    fn = sd._capi.HostProjectFn(rows)

    def desc(f=fn, length=D):
        return sd._capi.LevelHostProjectionC(f, None, 0, length, 0)

    def eyes(right, left):
        return sd.InterEyeDistanceNormalisation([str(i) for i in range(8)], [str(right)], [str(left)]).c()

    def train(proj, ld_=ld, norm=None, x=cur, p=P, x_next=nxt, chunk=n):
        return lib.sd_train_level_host_projected(ctx.h, None, C.byref(proj), ptr(x), ptr(gt), n, p, n, C.byref(norm) if norm else None,
                                                 None, 0, C.byref(reg), 0, ptr(buf), ld_, chunk, ptr(X), ptr(x_next), None)

    def apply(proj, ld_=ld, norm=None, x_next=nxt, chunk=n):
        return lib.sd_apply_level_host_projected(ctx.h, C.byref(proj), ptr(cur), n, P, C.byref(norm) if norm else None, None, 0, ptr(X),
                                                 ptr(buf), ld_, chunk, ptr(x_next))

    launches = ctx.launches()
    assert train(desc(f=sd._capi.HostProjectFn())) == 1 and apply(desc(f=sd._capi.HostProjectFn())) == 1      # no callback
    assert "needs a callback" in lib.sd_last_error(ctx.h).decode()
    assert train(desc(length=0)) == 1 and apply(desc(length=0)) == 1
    assert train(desc(), ld_=D + P - 1) == 1 and apply(desc(), ld_=D - 1) == 1
    assert train(desc(), x_next=cur) == 1 and apply(desc(), x_next=cur) == 1
    assert train(desc(), chunk=0) == 1 and apply(desc(), chunk=0) == 1
    odd = torch.from_numpy(np.ascontiguousarray(np.tile(x0[:, :1], (1, 7)))).cuda()                  # P = 7: no [x.., y..] rows
    assert train(desc(), norm=eyes(0, 1), x=odd, p=7) == 1
    assert "even P" in lib.sd_last_error(ctx.h).decode()
    assert train(desc(), norm=eyes(0, 3)) == 1 and apply(desc(), norm=eyes(3, 1)) == 1                 # eye index >= P / 2 = 3
    assert ctx.launches() == launches and not calls                      # refused before any work was queued
    ctx.sync()
    assert bool((X == 7.0).all()) and bool((nxt == 7.0).all())
    # the same descriptor with a valid normalisation of P = 6 trains
    assert train(desc(), norm=eyes(0, 2)) == 0 and calls == [0]          # one chunk: projected once

"""Multi-GPU training path on hardware (SURVEY.md 8e, 8f/f3): the C ABI's communicator, the band-packed Gram exchange and the
distributed blocked Cholesky (sd_learn_dist / sd_solve_gram_dist) against the one-GPU solve of the same rows.

  * one rank: runs on any GPU box (the communicator degenerates, the code path is the distributed one's host logic);
  * two ranks: needs two GPUs (`python -m pytest tests/test_gpu_multi.py -m gpu` on a box with two); skipped otherwise.

Bars: X(2 ranks) vs X(1 rank) <= 1e-5 relative (they differ only by the summation order of the two partial Gram matrices);
every rank holds the same X bit for bit; weights vs the float64 solve of the oracle's system <= 1e-4."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _system(n, d, m, seed):
    """HOG-like rows: non-negative, clamped at 0.2, block structure, bias column of ones (as tests/test_gpu_regressor.py)."""
    rng = np.random.default_rng(seed)
    A = np.minimum(np.abs(rng.standard_normal((n, d))).astype(np.float32) * 0.08, 0.2).astype(np.float32)
    A[:, ::7] *= 0.25
    A[:, -1] = 1.0
    B = (0.05 * rng.standard_normal((n, m))).astype(np.float32)
    return A, B


def _truth(A, B, lam_param):
    A64 = A.astype(np.float64)
    G = A64.T @ A64
    lam = np.float32(lam_param) * np.float32(np.linalg.norm(G.astype(np.float32).astype(np.float64))) / np.float32(A.shape[0])
    reg = np.eye(G.shape[0]) * float(lam)
    reg[-1, -1] = 0.0
    return np.linalg.solve(G + reg, A64.T @ B.astype(np.float64)), float(lam)


def _learn_dist(sd, ctx, comm_h, A_local, B_local, n_global, D, M, distributed_solve, regulariser=None):
    """The training step of the shells / the Python mirror on this rank's rows: centre (global means), Gram, exchange, solve."""
    import torch
    from superviseddescent_b200 import _capi
    dev = f"cuda:{ctx.device}"
    ld = (D + M + 3) // 4 * 4
    ext = torch.zeros((max(A_local.shape[0], 1), ld), dtype=torch.float32, device=dev)
    if A_local.shape[0]:
        ext[:A_local.shape[0], :D] = torch.from_numpy(A_local).to(dev)
        ext[:A_local.shape[0], D:D + M] = torch.from_numpy(B_local).to(dev)
    X = torch.empty((D, M), dtype=torch.float32, device=dev)
    mu = torch.empty(D, dtype=torch.float32, device=dev)
    lam = C.c_float(0)
    reg = (regulariser or sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)).c()
    lib = _capi.lib()
    rc = lib.sd_centre_features(ctx.h, comm_h, C.c_void_p(ext.data_ptr()), C.c_int64(ld), A_local.shape[0], D, n_global, C.byref(reg), C.c_void_p(mu.data_ptr()))
    if not rc:
        rc = lib.sd_learn_centred(ctx.h, comm_h, C.c_void_p(ext.data_ptr()), C.c_int64(ld), C.c_void_p(ext.data_ptr() + 4 * D), C.c_int64(ld),
                                  A_local.shape[0], D, M, C.byref(reg), n_global, int(distributed_solve), C.c_void_p(mu.data_ptr()),
                                  C.c_void_p(X.data_ptr()), None, C.byref(lam))
    if rc:
        raise RuntimeError(lib.sd_last_error(ctx.h).decode())
    return X.cpu().numpy(), lam.value


def test_one_rank_communicator_equals_plain_learn(sd):
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    A, B = _system(1500, 1301, 44, 11)               # 6 panels of 256 rows, ragged last one
    lr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False))
    lr.learn(A, B)
    X1 = lr.x.cpu().numpy()
    comm = C.c_void_p()
    assert _capi.lib().sd_comm_create(ctx.h, None, 0, 1, C.byref(comm)) == 0
    try:
        for ds in (0, 1):
            X, lam = _learn_dist(sd, ctx, comm, A, B, A.shape[0], A.shape[1], B.shape[1], ds)
            assert np.array_equal(X, X1)
    finally:
        _capi.lib().sd_comm_destroy(comm)
    Xt, lam_t = _truth(A, B, 1.5)
    e = rel_err(X1, Xt)
    print(f"one rank: weights vs float64 {e:.2e}")
    assert e <= 1e-4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_main(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # bootstrap only: carries the NCCL id
    from superviseddescent_b200 import api as sd
    from superviseddescent_b200 import parallel
    ctx = sd.Context(rank)
    comm = parallel.Communicator(ctx)
    res = {}
    for name, (n, d, m) in {"small": (900, 700, 44), "panels": (3001, 2900, 44)}.items():
        A, B = _system(n, d, m, 21)
        b, e = parallel.shard_range(n, world, rank)
        n_global = comm.sum_int(e - b)
        assert n_global == n
        for ds in (0, 1, 2):
            X, lam = _learn_dist(sd, ctx, comm.h, A[b:e], B[b:e], n_global, d, m, ds)
            res[(name, ds)] = (X, lam)
            res[(name, ds, "its")] = ctx.solver_iterations()
    # a system CG cannot finish (hardly regularised, condition number ~1e4): route 2 must hand over to the factorisation, which
    # needs the part of the matrix the CG route had not prepared on this rank
    A, B = _system(3001, 2900, 44, 21)
    b, e = parallel.shard_range(3001, world, rank)
    weak = sd.Regulariser(sd.RegularisationType.Manual, 1e-4, False)
    for ds in (0, 2):
        X, lam = _learn_dist(sd, ctx, comm.h, A[b:e], B[b:e], 3001, 2900, 44, ds, weak)
        res[("fallback", ds)] = (X, ctx.solver_iterations())
    # the whole cascade: two levels of HOG training on sharded samples, through the Python mirror
    import synth
    from oracle import oracle as O       # test infrastructure: only for the model's ids / mean
    om = O.Model(os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin"))
    n, size = 1200, 96
    images = synth.smooth_images(n, size, size, seed=77)
    rng = np.random.default_rng(77)
    box = np.array([5, 5, 86, 86])
    x0 = np.tile(O.align_mean(om.mean, box), (n, 1)).astype(np.float32)
    x_gt = np.stack([O.align_mean(om.mean, box, 1.0 + rng.normal(0, 0.04), 1.0 + rng.normal(0, 0.04), rng.normal(0, 0.04), rng.normal(0, 0.04))
                     for _ in range(n)]).astype(np.float32)
    hps = [sd.HoGParam(1, 3, 8, 4, 1.0), sd.HoGParam(1, 3, 6, 4, 0.5)]
    b, e = parallel.shard_range(n, world, rank)
    norm = sd.InterEyeDistanceNormalisation(om.landmark_ids, om.right_ids, om.left_ids)
    for ds in (False, True):
        ht = sd.HogTransform(images[b:e], hps, om.landmark_ids, om.right_ids, om.left_ids, ctx)
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), ctx) for _ in hps]
        sdo = sd.SupervisedDescentOptimiser(regs, norm, ctx)
        seen = []
        xf = sdo.train(x_gt[b:e], x0[b:e], None, ht, lambda cur: seen.append(cur.shape[0]), comm=comm, distributed_solve=ds)
        assert seen == [n, n]                            # the callback sees all rows (superviseddescent.hpp:217)
        res[("cascade", int(ds))] = ([r.x.cpu().numpy() for r in regs], xf.cpu().numpy())
    if rank == 0:                                        # the same rows on ONE GPU
        for name, (n_, d, m) in {"small": (900, 700, 44), "panels": (3001, 2900, 44)}.items():
            A, B = _system(n_, d, m, 21)
            lr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), ctx)
            lr.learn(A, B)
            res[(name, "single")] = (lr.x.cpu().numpy(), lr.last_lambda)
            res[(name, "truth")] = _truth(A, B, 1.5)
        ht = sd.HogTransform(images, hps, om.landmark_ids, om.right_ids, om.left_ids, ctx)
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), ctx) for _ in hps]
        sdo = sd.SupervisedDescentOptimiser(regs, norm, ctx)
        xf = sdo.train(x_gt, x0, None, ht)
        res[("cascade", "single")] = ([r.x.cpu().numpy() for r in regs], xf.cpu().numpy())
    out.put((rank, res))
    comm.close()
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_match_one_rank():
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    world = 2
    mpc = mp.get_context("spawn")
    out = mpc.Queue()
    port = _free_port()
    procs = [mpc.Process(target=_rank_main, args=(r, world, port, out)) for r in range(world)]
    for p in procs:
        p.start()
    results = dict(out.get(timeout=900) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    r0, r1 = results[0], results[1]
    for name in ("small", "panels"):
        Xs, lam_s = r0[(name, "single")]
        Xt, lam_t = r0[(name, "truth")]
        for ds in (0, 1, 2):
            X0, lam0 = r0[(name, ds)]
            X1, lam1 = r1[(name, ds)]
            assert np.array_equal(X0, X1) and lam0 == lam1                  # every rank ends with the same model
            e_single, e_truth = rel_err(X0, Xs), rel_err(X0, Xt)
            print(f"{name} distributed_solve={ds}: X(2 ranks) vs X(1 rank) {e_single:.2e}; vs float64 {e_truth:.2e}; lambda {lam0:.6g} / {lam_s:.6g} / {lam_t:.6g}; "
                  f"CG iterations {r0[(name, ds, 'its')]}")
            assert r0[(name, ds, "its")] > 0 if ds == 2 else r0[(name, ds, "its")] == 0    # converged CG / CG not tried
            assert e_single <= (1e-5 if ds < 2 else 2e-5)                   # CG stops at a relative residual of 2e-6
            assert e_truth <= 1e-4
            assert abs(lam0 - lam_s) <= 1e-6 * lam_s
    for r in (r0, r1):
        (Xa, its_a), (Xb, its_b) = r[("fallback", 0)], r[("fallback", 2)]
        print(f"fall-back: CG gave up after {-its_b} iterations; factorisation result identical to route 0: {np.array_equal(Xa, Xb)}")
        assert its_a == 0 and its_b < 0
        assert np.array_equal(Xa, Xb)                                       # the replicated factorisation of the same matrix
    assert np.array_equal(r0[("fallback", 2)][0], r1[("fallback", 2)][0])
    Ws, xs = r0[("cascade", "single")]
    n = xs.shape[0]
    for ds in (0, 1):
        W0, xa = r0[("cascade", ds)]
        W1, xb = r1[("cascade", ds)]
        x2 = np.concatenate([xa, xb])                                       # rank 0 holds the first shard
        assert x2.shape[0] == n
        for lvl in range(len(Ws)):
            assert np.array_equal(W0[lvl], W1[lvl])
            e = rel_err(W0[lvl], Ws[lvl])
            print(f"cascade distributed_solve={ds} level {lvl}: weights(2 ranks) vs weights(1 rank) {e:.2e}")
            assert e <= 1e-4          # level 1 starts from landmarks that already differ by rounding: crop centres may move by a pixel
        print(f"cascade distributed_solve={ds}: final landmarks 2 ranks vs 1 rank {rel_err(x2, xs):.2e}")
        assert np.mean(np.max(np.abs(x2 - xs), axis=1) <= 1e-3) >= 0.99

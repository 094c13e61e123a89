"""The rank diagnostic at any feature dimension (blocked pivoted Cholesky, superviseddescent_b200/csrc/sd_rank.cu) and from the
cascade's train().

Truth: LAPACK dpstrf on the float64 Gram with the device's cut, tol = eps_f32 * D * max(diag).  Where the inputs are synthetic,
the test first asserts that no float64 pivot lies within a factor of 10 of the cut, so the float32 device rank must equal it;
on real HOG features it may differ by the number of float64 pivots within a factor of 2 of the cut."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.linalg import lapack

import synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS_F32 = float(np.finfo(np.float32).eps)


def _gram64(A):
    """float64 Gram of float32 rows (computed on the device in float64: test infrastructure, not the product path)."""
    import torch
    t = torch.as_tensor(A, device="cuda").double()
    return (t.T @ t).cpu().numpy()


def _dpstrf_rank(G, tol):
    _, _, rank, info = lapack.dpstrf(np.asfortranarray(G), tol=tol, lower=0)
    assert info in (0, 1)
    return int(rank)


def _cut(G):
    return EPS_F32 * G.shape[0] * float(np.max(np.diag(G)))


def _pivots_near_cut(G, factor):
    """float64 pivots in (cut / factor, cut * factor]"""
    c = _cut(G)
    return _dpstrf_rank(G, c / factor) - _dpstrf_rank(G, c * factor)


def _rank_revealing(sd, A, lam, M=2):
    """sd_learn_rank_revealing on the rows A (float32, N x D); returns (rank, status)."""
    import torch
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    At = torch.as_tensor(A, device="cuda").contiguous()
    N, D = At.shape
    B = torch.ones((N, M), dtype=torch.float32, device="cuda")
    X = torch.empty((D, M), dtype=torch.float32, device="cuda")
    reg = sd.Regulariser(sd.RegularisationType.Manual, lam, True).c()
    lam_out, rank = C.c_float(0), C.c_int(-2)
    rc = _capi.lib().sd_learn_rank_revealing(ctx.h, C.c_void_p(At.data_ptr()), C.c_int64(D), C.c_void_p(B.data_ptr()), C.c_int64(M),
                                             N, D, M, C.byref(reg), C.c_void_p(X.data_ptr()), C.byref(lam_out), C.byref(rank))
    assert rc in (0, 5), _capi.lib().sd_last_error(ctx.h).decode()      # 5: the factorisation of a singular system stopped
    return rank.value, rc


@pytest.mark.parametrize("D", [4097, 4224, 5000, 8801])
def test_rank_revealing_beyond_the_one_cta_range(sd, D):
    rng = np.random.default_rng(D)
    A = rng.standard_normal((2 * D, D)).astype(np.float32)
    A[:, -1] = 1.0
    A[:, 10:50] = A[:, 100:140]                                        # 40 duplicated columns
    r0, _ = _rank_revealing(sd, A, 0.0)
    r0b, _ = _rank_revealing(sd, A, 0.0)
    assert r0 == D - 40 and r0b == r0                                  # exact, and the same on a second call
    assert sd.default_context().last_rank() == r0
    # with lambda > 0 a duplicate's pivot is about 2 lambda: regular once that is well above the cut (eps * D * 2D here)
    assert _rank_revealing(sd, A, 0.02 * D)[0] == D
    # fewer samples than features, rows from 256 latent factors (unit variance) and the bias: the rank float64 dpstrf finds at
    # the same cut
    L = (rng.standard_normal((D // 2, 256)) @ rng.standard_normal((256, D)) / 16.0).astype(np.float32)
    L[:, -1] = 1.0
    G = _gram64(L)
    assert _pivots_near_cut(G, 10.0) == 0, "the input has a float64 pivot within a factor of 10 of the cut"
    want = _dpstrf_rank(G, _cut(G))
    got, _ = _rank_revealing(sd, L, 0.0)
    print(f"D={D}: duplicated columns {r0}, low rank {got} (float64 {want})")
    assert got == want


def _hog_setup(oracle, golden, n, size, seed):
    om = oracle.Model(golden.model_path)
    images = synth.smooth_images(n, size, size, seed=seed)
    rng = np.random.default_rng(seed)
    box = np.array([5, 5, size - 10, size - 10])
    x0 = np.tile(oracle.align_mean(om.mean, box), (n, 1)).astype(np.float32)
    x_gt = np.stack([oracle.align_mean(om.mean, box, 1.0 + rng.normal(0, 0.04), 1.0 + rng.normal(0, 0.04), rng.normal(0, 0.04), rng.normal(0, 0.04))
                     for _ in range(n)]).astype(np.float32)
    return om, images, x0, x_gt


def test_rank_of_hog_features(sd, oracle, golden):
    """22 landmarks, K = 4, 5 x 5 cells: D = 8801 real features of N < D synthetic frames, lambda = 0."""
    om, images, x0, _ = _hog_setup(oracle, golden, 3000, 96, 7)
    ht = sd.HogTransform(images, [sd.HoGParam(1, 5, 6, 4, 0.25)], om.landmark_ids, om.right_ids, om.left_ids)
    A = ht(x0, 0).cpu().numpy()
    assert A.shape == (3000, 8801)
    G = _gram64(A)
    want = _dpstrf_rank(G, _cut(G))
    band = _pivots_near_cut(G, 2.0)
    got, _ = _rank_revealing(sd, A, 0.0)
    print(f"HOG features: rank {got}, float64 {want}, float64 pivots within a factor of 2 of the cut {band}")
    assert abs(got - want) <= band


def test_train_with_qr_solver_reports_rank(sd, oracle, golden, capsys):
    om, images, x0, x_gt = _hog_setup(oracle, golden, 600, 96, 2024)
    hps = [sd.HoGParam(1, 3, 8, 4, 1.0), sd.HoGParam(1, 3, 6, 4, 0.5)]          # D = 22*9*16+1 = 3169
    norm = sd.InterEyeDistanceNormalisation(om.landmark_ids, om.right_ids, om.left_ids)
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)
    results = {}
    for name, solver in (("lu", sd.PartialPivLUSolver), ("qr", sd.ColPivHouseholderQRSolver)):
        ht = sd.HogTransform(images, hps, om.landmark_ids, om.right_ids, om.left_ids)
        sdo = sd.SupervisedDescentOptimiser([sd.LinearRegressor(reg, solver=solver()) for _ in hps], norm)
        xf = sdo.train(x_gt, x0, None, ht).cpu().numpy()
        results[name] = (xf, [r.x.cpu().numpy() for r in sdo.regressors], [r.last_rank for r in sdo.regressors])
    assert results["qr"][2] == [3169, 3169]
    assert results["lu"][2] == [None, None]
    assert np.array_equal(results["qr"][0], results["lu"][0])          # the diagnostic does not touch the solve
    for a, b in zip(results["qr"][1], results["lu"][1]):
        assert np.array_equal(a, b)
    sd.LinearRegressor(reg).learn(ht(x0, 0), x_gt - x0)               # the switch is off again after the QR levels
    assert sd.default_context().last_rank() == -1
    # no regularisation and fewer samples than features: the message, then SdError with the rank of the centred system
    ht = sd.HogTransform(images, hps, om.landmark_ids, om.right_ids, om.left_ids)
    qr = sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.Manual, 0.0, False), solver=sd.ColPivHouseholderQRSolver())
    sdo = sd.SupervisedDescentOptimiser([qr], norm)
    capsys.readouterr()
    with pytest.raises(sd.SdError) as e:
        sdo.train(x_gt, x0, None, ht)
    r = qr.last_rank
    assert 0 < r < 3169
    assert f"(The rank is {r}, full rank would be 3169)" in str(e.value)
    assert f"(The rank is {r}, full rank would be 3169). Increase lambda." in capsys.readouterr().out
    A = ht(x0, 0).cpu().numpy().astype(np.float64)
    A[:, :-1] -= A[:, :-1].mean(axis=0)                                # the centred rows the train solves on
    G = A.T @ A
    want, band = _dpstrf_rank(G, _cut(G)), _pivots_near_cut(G, 2.0)
    print(f"train, lambda = 0: rank {r}, float64 of the centred system {want}, pivots within a factor of 2 of the cut {band}")
    assert abs(r - want) <= band


def _two_rank_main(rank, world, port, out):
    import sys
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # bootstrap only: carries the NCCL id
    from superviseddescent_b200 import _capi, api as sd, parallel
    ctx = sd.Context(rank)
    comm = parallel.Communicator(ctx)
    rng = np.random.default_rng(5)
    n, D, M = 3000, 2900, 8
    A = rng.standard_normal((n, D)).astype(np.float32)
    A[:, -1] = 1.0
    b, e = parallel.shard_range(n, world, rank)
    ld = (D + M + 3) // 4 * 4
    ext = torch.zeros((e - b, ld), dtype=torch.float32, device=f"cuda:{rank}")
    ext[:, :D] = torch.from_numpy(A[b:e]).to(ext.device)
    ext[:, D:D + M] = 1.0
    X = torch.empty((D, M), dtype=torch.float32, device=ext.device)
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    res = {}
    ctx.set_rank_diagnostic(True)
    for ds in (0, 1, 2):
        _capi.lib().sd_learn_dist(ctx.h, comm.h, C.c_void_p(ext.data_ptr()), C.c_int64(ld), C.c_void_p(ext.data_ptr() + 4 * D), C.c_int64(ld),
                                  e - b, D, M, C.byref(reg), n, ds, C.c_void_p(X.data_ptr()), None)
        res[ds] = ctx.last_rank()
    ctx.set_rank_diagnostic(False)
    if rank == 0:
        one = sd.Context(rank)
        one.set_rank_diagnostic(True)
        ext1 = torch.zeros((n, ld), dtype=torch.float32, device=ext.device)
        ext1[:, :D] = torch.from_numpy(A).to(ext.device)
        ext1[:, D:D + M] = 1.0
        _capi.lib().sd_learn(one.h, C.c_void_p(ext1.data_ptr()), C.c_int64(ld), C.c_void_p(ext1.data_ptr() + 4 * D), C.c_int64(ld),
                             n, D, M, C.byref(reg), C.c_void_p(X.data_ptr()), None)
        res["single"] = one.last_rank()
        one.close()
    out.put((rank, res))
    comm.close()
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_report_the_one_gpu_rank():
    import socket
    import torch
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    mpc = mp.get_context("spawn")
    out = mpc.Queue()
    procs = [mpc.Process(target=_two_rank_main, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    results = dict(out.get(timeout=900) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    single = results[0]["single"]
    assert single == 2900
    for r in (0, 1):
        assert results[r][0] == single and results[r][2] == single    # replicated and shared-CG routes: the one-GPU rank
        assert results[r][1] == -1                                     # distributed factorisation: not computed

"""Training and testing HogTransform levels in chunks of rows (sd_train_level, sd_apply_level, sd_level_chunk_rows).

One chunk must be the one-shot level bit for bit: a helper here replays that call sequence through the C ABI (sd_hog_batch,
sd_subtract_templates, sd_cascade_targets, sd_centre_features, sd_learn_centred, sd_cascade_update).  Several chunks must meet
the float64 bars of test_gpu_train.py and stay within 1e-5 of one chunk."""
import ctypes as C
import os
import socket
import sys

import numpy as np
import pytest

import synth
from conftest import rel_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HPS = [(1, 3, 8, 4, 1.0), (1, 3, 6, 4, 0.5)]           # D = 22*9*16+1 = 3169
SMALL = [(1, 1, 8, 2, 1.0)]                              # D = 22*10+1 = 221: reference-order LU, no shift


def _fixture(om, O, n=900, size=96, seed=2024):
    images = synth.smooth_images(n, size, size, seed=seed)
    rng = np.random.default_rng(seed)
    box = np.array([5, 5, 86, 86])
    x0 = np.tile(O.align_mean(om.mean, box), (n, 1)).astype(np.float32)
    x_gt = np.stack([O.align_mean(om.mean, box, 1.0 + rng.normal(0, 0.04), 1.0 + rng.normal(0, 0.04), rng.normal(0, 0.04), rng.normal(0, 0.04))
                     for _ in range(n)]).astype(np.float32)
    return images, x0, x_gt


def _optimiser(sd, om, levels, solver=None):
    regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), solver=solver) for _ in range(levels)]
    return sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(om.landmark_ids, om.right_ids, om.left_ids))


def _one_shot_train(sd, ctx, ht, x_gt, x0, n_levels, qr=False, tmpl=None):
    """The one-shot level, call by call: all N feature rows [A | b] resident, centred in place, learned, updated."""
    import torch
    lib = sd._capi.lib()
    ptr = sd._capi.ptr
    dev = f"cuda:{ctx.device}"
    cur = torch.from_numpy(x0).to(dev)
    gt = torch.from_numpy(x_gt).to(dev)
    n, P = cur.shape
    norm = eyes = ht.norm.c()                                # the optimiser normalises with the HogTransform's eyes
    if tmpl is not None:
        tmpl = torch.from_numpy(tmpl).to(dev)
    out = []
    for level in range(n_levels):
        D = ht.feature_length(level)
        ld = (D + P + 3) // 4 * 4
        A = torch.empty((n, ld), dtype=torch.float32, device=dev)
        reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
        assert lib.sd_hog_batch(ctx.h, C.byref(ht.batch()), None, ptr(cur), C.c_int64(P), n, P // 2, C.byref(eyes),
                                C.byref(ht.hog_params[level]), ptr(A), C.c_int64(ld)) == 0
        if tmpl is not None:
            assert lib.sd_subtract_templates(ctx.h, ptr(A), C.c_int64(ld), ptr(tmpl), C.c_int64(tmpl.stride(0)), n, D) == 0
        assert lib.sd_cascade_targets(ctx.h, ptr(cur), ptr(gt), n, P, C.byref(norm), ptr(A[:, D:]), C.c_int64(ld)) == 0
        mu = torch.empty(D, dtype=torch.float32, device=dev)
        X = torch.empty((D, P), dtype=torch.float32, device=dev)
        Xc = torch.empty((D, P), dtype=torch.float32, device=dev)
        lam = C.c_float(0)
        assert lib.sd_centre_features(ctx.h, None, ptr(A), C.c_int64(ld), n, D, n, C.byref(reg), ptr(mu)) == 0
        if qr:
            ctx.set_rank_diagnostic(True)
        assert lib.sd_learn_centred(ctx.h, None, ptr(A), C.c_int64(ld), ptr(A[:, D:]), C.c_int64(ld), n, D, P, C.byref(reg), n, 0,
                                    ptr(mu), ptr(X), ptr(Xc), C.byref(lam)) == 0
        rank = ctx.last_rank()
        ctx.set_rank_diagnostic(False)
        nxt = torch.empty_like(cur)
        assert lib.sd_cascade_update(ctx.h, ptr(A), C.c_int64(ld), n, D, ptr(Xc), P, ptr(cur), C.byref(norm), ptr(nxt)) == 0
        out.append((X.cpu().numpy(), lam.value, rank))
        cur = nxt
    ctx.sync()
    return out, cur.cpu().numpy()


def _one_shot_test(sd, ctx, ht, regs, x0):
    import torch
    lib = sd._capi.lib()
    ptr = sd._capi.ptr
    cur = torch.from_numpy(x0).to(f"cuda:{ctx.device}")
    n, P = cur.shape
    norm = ht.norm.c()
    for level, r in enumerate(regs):
        D = ht.feature_length(level)
        ld = (D + 3) // 4 * 4
        A = torch.empty((n, ld), dtype=torch.float32, device=cur.device)
        assert lib.sd_hog_batch(ctx.h, C.byref(ht.batch()), None, ptr(cur), C.c_int64(P), n, P // 2, C.byref(norm),
                                C.byref(ht.hog_params[level]), ptr(A), C.c_int64(ld)) == 0
        nxt = torch.empty_like(cur)
        assert lib.sd_cascade_update(ctx.h, ptr(A), C.c_int64(ld), n, D, ptr(r.x), P, ptr(cur), C.byref(norm), ptr(nxt)) == 0
        cur = nxt
    return cur.cpu().numpy()


@pytest.fixture(scope="module")
def setup(sd, oracle, golden):
    om = oracle.Model(golden.model_path)
    images, x0, x_gt = _fixture(om, oracle)
    return om, images, x0, x_gt


@pytest.mark.parametrize("case", ["matrixnorm", "small", "qr"])
def test_one_chunk_is_the_one_shot_level(sd, setup, case):
    om, images, x0, x_gt = setup
    ctx = sd.default_context()
    hps = [sd.HoGParam(*h) for h in (SMALL if case == "small" else HPS)]
    ht = sd.HogTransform(images, hps, om.landmark_ids, om.right_ids, om.left_ids)
    qr = case == "qr"
    sdo = _optimiser(sd, om, len(hps), sd.ColPivHouseholderQRSolver() if qr else None)
    got = sdo.train(x_gt, x0, None, ht).cpu().numpy()
    want, want_x = _one_shot_train(sd, ctx, ht, x_gt, x0, len(hps), qr=qr)
    assert np.array_equal(got, want_x)
    for r, (X, lam, rank) in zip(sdo.regressors, want):
        assert np.array_equal(r.x.cpu().numpy(), X) and r.last_lambda == lam
        if qr:
            assert r.last_rank == rank == X.shape[0]
    assert np.array_equal(sdo.test(x0, None, ht).cpu().numpy(), _one_shot_test(sd, ctx, ht, sdo.regressors, x0))
    # a chunked test() computes every row as the one-shot level does
    assert np.array_equal(sdo.test(x0, None, ht, rows_per_chunk=256).cpu().numpy(), _one_shot_test(sd, ctx, ht, sdo.regressors, x0))


def test_one_chunk_with_templates_is_the_one_shot_level(sd, setup):
    om, images, x0, x_gt = setup
    ctx = sd.default_context()
    ht = sd.HogTransform(images, [sd.HoGParam(*HPS[0])], om.landmark_ids, om.right_ids, om.left_ids)
    D = ht.feature_length(0)
    tmpl = np.random.default_rng(1).uniform(0, 0.01, (x0.shape[0], D)).astype(np.float32)
    tmpl[:, -1] = 0.0                                       # the bias column stays all ones
    sdo = _optimiser(sd, om, 1)
    got = sdo.train(x_gt, x0, tmpl, ht, rows_per_chunk=300).cpu().numpy()      # templates take one chunk whatever is asked
    want, want_x = _one_shot_train(sd, ctx, ht, x_gt, x0, 1, tmpl=tmpl)
    assert np.array_equal(got, want_x) and np.array_equal(sdo.regressors[0].x.cpu().numpy(), want[0][0])


_TRUTH = {}


def _truth(oracle, om, images, cur, x_gt, level):
    from test_gpu_train import _truth_level
    key = (level, cur.tobytes())
    if key not in _TRUTH:
        _TRUTH[key] = _truth_level(oracle, om, images, cur, x_gt, oracle.HogParam(*HPS[level]), 1.5)
    return _TRUTH[key]


@pytest.mark.parametrize("mode", [0, 2])
@pytest.mark.parametrize("rows", [256, 300, 899])
def test_several_chunks_meet_the_float64_bars(sd, oracle, setup, rows, mode):
    om, images, x0, x_gt = setup
    ctx = sd.default_context()
    ctx.set_gram_mode(mode)
    try:
        cur = x0
        for level in range(2):
            _, X_ref, lam_ref, nxt_ref = _truth(oracle, om, images, cur, x_gt, level)
            ht = sd.HogTransform(images, [sd.HoGParam(*HPS[level])], om.landmark_ids, om.right_ids, om.left_ids)
            one, many = _optimiser(sd, om, 1), _optimiser(sd, om, 1)
            one.train(x_gt, cur, None, ht)
            got = many.train(x_gt, cur, None, ht, rows_per_chunk=rows).cpu().numpy()
            X, X1 = many.regressors[0].x.cpu().numpy(), one.regressors[0].x.cpu().numpy()
            lam = many.regressors[0].last_lambda
            e_w, e_x, e_1 = rel_err(X, X_ref), rel_err(got, nxt_ref), rel_err(X, X1)
            print(f"rows {rows} mode {mode} level {level}: lambda {lam:.6g} vs {lam_ref:.6g}; weights vs float64 {e_w:.2e}, vs one chunk "
                  f"{e_1:.2e}; landmarks {e_x:.2e}")
            assert abs(lam - lam_ref) <= 2e-5 * lam_ref
            assert e_w <= 2e-5 and e_x <= 1e-4 and e_1 <= 1e-5
            cur = nxt_ref
    finally:
        ctx.set_gram_mode(0)


def test_chunked_qr_level_reports_the_rank_of_one_chunk(sd, setup):
    om, images, x0, x_gt = setup
    ht = sd.HogTransform(images, [sd.HoGParam(*HPS[0])], om.landmark_ids, om.right_ids, om.left_ids)
    ranks = []
    for rows in (None, 300):
        sdo = _optimiser(sd, om, 1, sd.ColPivHouseholderQRSolver())
        sdo.train(x_gt, x0, None, ht, rows_per_chunk=rows)
        ranks.append(sdo.regressors[0].last_rank)
    assert ranks[0] == ranks[1] == ht.feature_length(0)


def test_repeated_chunked_train_is_bit_identical(sd, setup):
    om, images, x0, x_gt = setup
    ht = sd.HogTransform(images, [sd.HoGParam(*h) for h in HPS], om.landmark_ids, om.right_ids, om.left_ids)
    runs = []
    for _ in range(2):
        sdo = _optimiser(sd, om, 2)
        xf = sdo.train(x_gt, x0, None, ht, rows_per_chunk=300).cpu().numpy()
        runs.append([r.x.cpu().numpy() for r in sdo.regressors] + [xf])
    assert all(np.array_equal(a, b) for a, b in zip(*runs))


def test_invalid_arguments_leave_the_outputs_unwritten(sd, setup):
    import torch
    om, images, x0, x_gt = setup
    ctx = sd.default_context()
    lib = sd._capi.lib()
    ptr = sd._capi.ptr
    ht = sd.HogTransform(images, [sd.HoGParam(*HPS[0])], om.landmark_ids, om.right_ids, om.left_ids)
    n, P = x0.shape
    D = ht.feature_length(0)
    ld = (D + P + 3) // 4 * 4
    cur, gt = torch.from_numpy(x0).cuda(), torch.from_numpy(x_gt).cuda()
    buf = torch.empty((n, ld), dtype=torch.float32, device="cuda")
    tmpl = torch.zeros((n, D), dtype=torch.float32, device="cuda")
    X = torch.full((D, P), 7.0, device="cuda")
    nxt = torch.full((n, P), 7.0, device="cuda")
    eyes, reg = ht.norm.c(), sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    frames = ht.level_frames(n)

    def train(chunk_rows=n, ld_=ld, t=None, x_next=nxt):
        return lib.sd_train_level(ctx.h, None, C.byref(frames), ptr(cur), ptr(gt), n, P // 2, C.c_int64(n), C.byref(eyes),
                                  C.byref(ht.hog_params[0]), C.byref(eyes), ptr(t), C.c_int64(D), C.byref(reg), 0, ptr(buf),
                                  C.c_int64(ld_), chunk_rows, ptr(X), ptr(x_next), None)

    def apply(chunk_rows=n, ld_=ld, x_next=nxt):
        return lib.sd_apply_level(ctx.h, C.byref(frames), ptr(cur), n, P // 2, C.byref(eyes), C.byref(ht.hog_params[0]),
                                  C.byref(eyes), None, C.c_int64(0), ptr(X), ptr(buf), C.c_int64(ld_), chunk_rows, ptr(x_next))

    launches = ctx.launches()
    assert train(chunk_rows=0) == 1 and apply(chunk_rows=0) == 1
    assert train(ld_=D + P - 1) == 1 and apply(ld_=D - 1) == 1
    assert train(chunk_rows=n - 1, t=tmpl) == 1
    assert train(x_next=cur) == 1 and apply(x_next=cur) == 1
    assert ctx.launches() == launches                        # refused before any work was queued
    ctx.sync()
    assert bool((X == 7.0).all()) and bool((nxt == 7.0).all())
    assert np.array_equal(cur.cpu().numpy(), x0)


def test_chunk_query_counts_host_staging(sd):
    ctx = sd.default_context()
    lib = sd._capi.lib()
    import torch
    hp = sd.HoGParam(1, 5, 6, 9, 1.0)
    D = lib.sd_hog_feature_length(22, C.byref(hp))
    assert D == 17051
    P = 44
    ld = (D + P + 3) // 4 * 4
    rows = C.c_int(0)
    assert lib.sd_level_chunk_rows(ctx.h, None, None, C.c_int64(10000), D, P, 0, C.c_size_t(0), C.byref(rows)) == 0
    assert rows.value == 10000
    free = torch.cuda.mem_get_info()[0]
    assert lib.sd_level_chunk_rows(ctx.h, None, None, C.c_int64(4000000), D, P, 0, C.c_size_t(free), C.byref(rows)) == 0
    print(f"D = {D}: {rows.value} rows of {ld * 4} bytes fit in {free / 1e9:.1f} GB")
    assert 0 < rows.value < 4000000
    assert rows.value * ld * 4 + (512 << 20) <= free
    # not even the minimal chunk fits (256 MB is below the reserve, whatever the context already holds): an error naming D
    assert lib.sd_level_chunk_rows(ctx.h, None, None, C.c_int64(4000000), D, P, 0, C.c_size_t(256 << 20), C.byref(rows)) == 2
    assert "17051" in lib.sd_last_error(ctx.h).decode()
    # host frames: the staging pair the level will hold is counted too (a fresh context holds none of it yet)
    fresh = sd.Context(ctx.device)
    img = np.zeros((16, 16), dtype=np.uint8)
    frames = sd.LevelFramesC(num_host_frames=1, stage_half_bytes=1 << 30)
    frames.host_frames = C.pointer(sd._host_frame(img)[0])
    dev_rows, host_rows = C.c_int(0), C.c_int(0)
    assert lib.sd_level_chunk_rows(fresh.h, None, None, C.c_int64(4000000), D, P, 0, C.c_size_t(free), C.byref(dev_rows)) == 0
    assert lib.sd_level_chunk_rows(fresh.h, None, C.byref(frames), C.c_int64(4000000), D, P, 0, C.c_size_t(free), C.byref(host_rows)) == 0
    pair_rows = (2 << 30) // (ld * 4 + P * 8)
    assert dev_rows.value - host_rows.value in (pair_rows, pair_rows + 1)


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
    from oracle import oracle as O
    from superviseddescent_b200 import api as sd
    from superviseddescent_b200 import parallel
    ctx = sd.Context(rank)
    comm = parallel.Communicator(ctx)
    om = O.Model(os.path.join(ROOT, "tests", "golden", "face_landmarks_model_rcr_22.bin"))
    images, x0, x_gt = _fixture(om, O)
    n = x0.shape[0]
    b, e = parallel.shard_range(n, world, rank)
    hps = [sd.HoGParam(*h) for h in HPS]
    res = {}
    for ds in (False, True, "cg"):
        ht = sd.HogTransform(images[b:e], hps, om.landmark_ids, om.right_ids, om.left_ids, ctx)
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), ctx) for _ in hps]
        sdo = sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(om.landmark_ids, om.right_ids, om.left_ids), ctx)
        sdo.train(x_gt[b:e], x0[b:e], None, ht, comm=comm, distributed_solve=ds, rows_per_chunk=128 + 64 * rank)
        res[str(ds)] = [r.x.cpu().numpy() for r in regs]
    if rank == 0:
        ht = sd.HogTransform(images, hps, om.landmark_ids, om.right_ids, om.left_ids, ctx)
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False), ctx) for _ in hps]
        sdo = sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(om.landmark_ids, om.right_ids, om.left_ids), ctx)
        sdo.train(x_gt, x0, None, ht)
        res["single"] = [r.x.cpu().numpy() for r in regs]
    out.put((rank, res))
    comm.close()
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_train_in_chunks():
    """Each rank trains its shard in chunks of its own size (the ranks' chunk counts differ) with routes 0, 1 and 2."""
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
    single = results[0]["single"]
    for ds in ("False", "True", "cg"):
        for level, (X0, X1, Xs) in enumerate(zip(results[0][ds], results[1][ds], single)):
            e = rel_err(X0, Xs)
            print(f"route {ds} level {level}: 2 ranks in chunks vs 1 GPU in one chunk {e:.2e}")
            assert np.array_equal(X0, X1) and e <= 1e-5

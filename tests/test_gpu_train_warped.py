"""Cascade levels on warped samples (sd_level_frames.d_sample_warp) against the same levels on materialised virtual frames: each
sample's V = cv2.warpAffine(grey frame, M, size, INTER_LINEAR | WARP_INVERSE_MAP) passed as a frame of its own.  X, lambda and
x_next must be bit for bit equal, on the device route and on the host route (grey and colour pinned frames: V is the warp of the
grey frame), in one chunk and in several; the host route's plan must never raise a miss.  HogTransform(warps=...) must train, test
and predict bit for bit as a transform over the copies."""
import ctypes as C

import cv2
import numpy as np
import pytest
import torch

import sample_warp_ref as SW
import test_gpu_train_mirrored as TM

pytestmark = pytest.mark.gpu

ADAPTIVE, REYE, LEYE = TM.ADAPTIVE, TM.REYE, TM.LEYE


def _grey(img):
    return img if img.ndim == 2 else cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)


@pytest.fixture(scope="module")
def setup(sd, golden):
    ctx = sd.default_context()
    m = sd.load_detection_model(golden.model_path, ctx)
    imgs = TM._images()
    frame, x0, x_gt = TM._samples(sd, m.get_mean())
    rng = np.random.default_rng(4)
    warps, sizes = [], []
    for k, f in enumerate(frame):
        w, h, _ = TM.SPECS[f]
        angle, scale = float(rng.uniform(-60, 60)), float(rng.uniform(0.8, 1.25))
        M = sd.rotation_warp((w / 2 + rng.uniform(-5, 5), h / 2 + rng.uniform(-5, 5)), angle, scale)
        if k % 5 == 4:
            M = np.array([[-1.0, 0, w - 1], [0, 1, 0]]) @ np.vstack([M, [0, 0, 1]])     # a reflection of the rotation
        warps.append(M)
        sizes.append((w + int(rng.integers(-10, 20)), h + int(rng.integers(-10, 20))))
    warps, sizes = np.stack(warps), np.array(sizes)
    inv = sd.invert_warp(warps)
    # landmarks in V's coordinates: the frame's samples carried through the inverse warp
    X0, XG = sd.warp_landmarks(x0, inv), sd.warp_landmarks(x_gt, inv)
    vs = [SW.materialise(_grey(imgs[f]), M, s) for f, M, s in zip(frame, warps, sizes)]
    return dict(ctx=ctx, ids=m.landmark_ids, imgs=imgs, vs=vs, frame=frame.astype(np.int32), warps=warps, sizes=sizes, X0=X0, XG=XG,
                own=TM._Set(sd, ctx, imgs), copies=TM._Set(sd, ctx, vs))


def _level(sd, S, which, host, chunk_rows, X=None):
    ctx, lib, ptr = S["ctx"], sd._capi.lib(), sd._capi.ptr
    n = len(S["X0"])
    idx = torch.from_numpy(S["frame"] if which == "own" else np.arange(n, dtype=np.int32)).cuda()
    frames = S[which].frames(sd, host, idx)
    table = sd._warp_table(S["warps"], S["sizes"], None, "cuda") if which == "own" else None
    frames.d_sample_warp = ptr(table)
    x0, xg = torch.from_numpy(S["X0"]).cuda(), torch.from_numpy(S["XG"]).cuda()
    P = x0.shape[1]
    p = sd.HoGParam(*ADAPTIVE)
    D = lib.sd_hog_feature_length(P // 2, C.byref(p))
    norm = sd.InterEyeDistanceNormalisation(S["ids"], REYE, LEYE).c()
    nxt = torch.full((n, P), 7.0, device="cuda")
    if X is None:
        ld = (D + P + 3) // 4 * 4
        buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
        Xo = torch.full((D, P), 7.0, device="cuda")
        lam = C.c_float(0)
        reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
        rc = lib.sd_train_level(ctx.h, None, C.byref(frames), ptr(x0), ptr(xg), n, P // 2, C.c_int64(n), C.byref(norm), C.byref(p),
                                C.byref(norm), None, C.c_int64(0), C.byref(reg), 0, ptr(buf), C.c_int64(ld), chunk_rows, ptr(Xo), ptr(nxt),
                                C.byref(lam))
        assert rc == 0, lib.sd_last_error(ctx.h).decode()
        ctx.sync()
        return Xo.cpu().numpy(), lam.value, nxt.cpu().numpy()
    ld = (D + 3) // 4 * 4
    buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
    Xd = torch.from_numpy(X).cuda()
    rc = lib.sd_apply_level(ctx.h, C.byref(frames), ptr(x0), n, P // 2, C.byref(norm), C.byref(p), C.byref(norm), None, C.c_int64(0),
                            ptr(Xd), ptr(buf), C.c_int64(ld), chunk_rows, ptr(nxt))
    assert rc == 0, lib.sd_last_error(ctx.h).decode()   # the host route fails the call on a planned-region miss
    ctx.sync()
    return nxt.cpu().numpy()


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("chunk", ["one", "several"])
def test_warped_levels_equal_materialised_levels(sd, setup, host, chunk):
    S = setup
    n = len(S["X0"])
    rows = n if chunk == "one" else 7
    got = _level(sd, S, "own", host, rows)
    want = _level(sd, S, "copies", host, rows)
    for k, what in ((0, "X"), (2, "x_next")):
        assert np.array_equal(TM._bits(got[k]), TM._bits(want[k])), what
    assert TM._bits(got[1]) == TM._bits(want[1]), "lambda"
    a = _level(sd, S, "own", host, rows, X=got[0])
    b = _level(sd, S, "copies", host, rows, X=got[0])
    assert np.array_equal(TM._bits(a), TM._bits(b)), "apply x_next"


@pytest.mark.parametrize("route", ["device", "host"])
def test_python_warped_transform_equals_copies(sd, setup, monkeypatch, route):
    S = setup
    hps = [sd.HoGParam(*ADAPTIVE), sd.HoGParam(1, 3, 6, 4, 0.8)]
    if route == "host":
        monkeypatch.setattr(sd, "DEVICE_FRAME_SHARE", 0.0)
        monkeypatch.setattr(sd, "HOST_STAGE_HALF", 64 << 10)
    own = sd.HogTransform(S["imgs"], hps, S["ids"], REYE, LEYE, image_index=S["frame"], warps=S["warps"], warp_sizes=S["sizes"])
    copies = sd.HogTransform(S["vs"], hps, S["ids"], REYE, LEYE)
    assert own.on_device() == (route == "device")
    res = []
    for h in (own, copies):
        regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)) for _ in hps]
        sdo = sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(S["ids"], REYE, LEYE))
        xt = sdo.train(S["XG"], S["X0"], None, h, rows_per_chunk=13)
        xs = sdo.test(S["X0"], None, h)
        xp = sdo.predict(S["X0"], None, h)
        res.append([r.x.cpu().numpy() for r in sdo.regressors] + [xt.cpu().numpy(), xs.cpu().numpy(), xp.cpu().numpy()])
    for k, (a, b) in enumerate(zip(*res)):
        assert np.array_equal(TM._bits(a), TM._bits(b)), k
    if route == "device":
        x = S["X0"]
        assert np.array_equal(TM._bits(own(x, 0).cpu().numpy()), TM._bits(copies(x, 0).cpu().numpy()))
        for a, b in zip(own.debug(x, 1), copies.debug(x, 1)):
            assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())


def test_python_warps_exclude_mirrored(sd, setup):
    S = setup
    n = len(S["frame"])
    with pytest.raises(ValueError):
        sd.HogTransform(S["imgs"], [sd.HoGParam(*ADAPTIVE)], S["ids"], REYE, LEYE, image_index=S["frame"], mirrored=[False] * n,
                        warps=S["warps"])

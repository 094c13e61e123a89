"""Cascade levels on frames that stay in host memory (sd_train_level, sd_apply_level with sd_level_frames.host_frames) and
HogTransform's frames shared by several samples.

The host route must give bit for bit what the device route gives on the same frames uploaded by sd_upload_frames: the HOG kernel
reads the same bytes, gathered from the planned regions instead of whole resident frames."""
import ctypes as C

import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

ADAPTIVE = (1, 3, 8, 4, 1.0)      # D = 22 * 9 * 16 + 1 = 3169
FIXED = (1, 3, 8, 4, 0.0)         # hog_eyes NULL: half = 3 * 4 = 12
REYE, LEYE = ["37", "40"], ["43", "46"]
SPECS = [(160, 120, 1), (200, 150, 3), (131, 97, 1), (176, 144, 3), (96, 96, 1), (150, 140, 3)]


def _round16(v):
    return (v + 15) // 16 * 16


def _pinned_frame(img, pad=0):
    """(h, w) or (h, w, 3) uint8 -> a pinned copy with a 16-byte aligned row pitch (+ pad bytes) and its array view"""
    import torch
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    pitch = ch * _round16(w) + pad
    t = torch.empty(h * pitch + 16, dtype=torch.uint8).pin_memory()
    off = (-t.data_ptr()) % 16
    a = t[off:off + h * pitch].numpy().reshape(h, pitch)
    a[:, :w * ch] = img.reshape(h, w * ch)
    view = np.lib.stride_tricks.as_strided(a, img.shape, (pitch, ch, 1) if ch == 3 else (pitch, 1))
    return t, view


def _images(seed=5):
    out = []
    for i, (w, h, ch) in enumerate(SPECS):
        g = synth.smooth_images(ch, h, w, seed=seed + i)
        out.append(g[0] if ch == 1 else np.ascontiguousarray(np.moveaxis(g, 0, -1)))
    return out


def _samples(sd, mean, n_frames, per_frame=11, seed=3):
    """per_frame samples of each frame in shuffled order, some hanging over the border, plus one entirely outside its frame"""
    rng = np.random.default_rng(seed)
    frame, x0, x_gt = [], [], []
    for f in range(n_frames):
        w, h, _ = SPECS[f]
        s = min(w, h) * 3 // 4
        for k in range(per_frame):
            bx = int(rng.integers(-s // 3, w - s + s // 3)) if k % 4 == 3 else (w - s) // 2 + int(rng.integers(-4, 5))
            by = int(rng.integers(-s // 3, h - s + s // 3)) if k % 4 == 3 else (h - s) // 2 + int(rng.integers(-4, 5))
            box = (bx, by, s, s)
            x_gt.append(sd.align_mean(mean, box))
            x0.append(sd.align_mean(mean, box, 1 + rng.normal(0, 0.04), 1 + rng.normal(0, 0.04), rng.normal(0, 0.04), rng.normal(0, 0.04)))
            frame.append(f)
    x_gt.append(sd.align_mean(mean, (-900, -900, 80, 80)))       # every patch outside frame 2
    x0.append(x_gt[-1].copy())
    frame.append(2)
    order = rng.permutation(len(frame))
    return (np.asarray(frame, dtype=np.int32)[order], np.asarray(x0, dtype=np.float32)[order],
            np.asarray(x_gt, dtype=np.float32)[order])


@pytest.fixture(scope="module")
def setup(sd, golden):
    import torch
    ctx = sd.default_context()
    m = sd.load_detection_model(golden.model_path, ctx)
    ids = m.landmark_ids
    imgs = _images()
    pinned = [_pinned_frame(img, pad=16 * (i % 2)) for i, img in enumerate(imgs)]
    frames, x0, x_gt = _samples(sd, m.get_mean(), len(imgs))
    recs = [sd._host_frame(v)[0] for _, v in pinned]
    table = (sd.HostFrameC * len(recs))(*recs)
    nbytes = C.c_size_t(0)
    lib = sd._capi.lib()
    assert lib.sd_upload_frames(ctx.h, table, len(recs), None, C.byref(nbytes), None) == 0
    dbuf = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
    ib = sd.ImageBatchC()
    assert lib.sd_upload_frames(ctx.h, table, len(recs), sd._capi.ptr(dbuf), C.byref(nbytes), C.byref(ib)) == 0
    return dict(ctx=ctx, ids=ids, imgs=imgs, pinned=pinned, table=table, nf=len(recs), ib=ib, dbuf=dbuf, frames=frames, x0=x0, x_gt=x_gt)


def _eyes(sd, ids):
    return sd.InterEyeDistanceNormalisation(ids, REYE, LEYE).c()


def _frames(sd, S, host, idx, stage_half=0, table=None):
    """the sd_level_frames of the setup's frames: host frames (table, default the setup's) or the uploaded batch"""
    f = sd.LevelFramesC(d_sample_frame=sd._capi.ptr(idx), stage_half_bytes=stage_half)
    if host:
        f.host_frames, f.num_host_frames = table if table is not None else S["table"], S["nf"]
    else:
        f.images = C.pointer(S["ib"])
    return f


def _train(sd, S, hp, host, chunk_rows, stage_half=0, eyes_on=True, rows=None):
    """one training level on the samples `rows` (default all) of the setup; rows given: sample i reads frame i (index NULL)"""
    import torch
    ctx, lib, ptr = S["ctx"], sd._capi.lib(), sd._capi.ptr
    sel = slice(None) if rows is None else rows
    x0, xg = torch.from_numpy(S["x0"][sel]).cuda(), torch.from_numpy(S["x_gt"][sel]).cuda()
    idx = torch.from_numpy(S["frames"]).cuda() if rows is None else None
    n, P = x0.shape
    p = sd.HoGParam(*hp)
    D = lib.sd_hog_feature_length(P // 2, C.byref(p))
    ld = (D + P + 3) // 4 * 4
    buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
    X = torch.full((D, P), 7.0, device="cuda")
    nxt = torch.full((n, P), 7.0, device="cuda")
    lam = C.c_float(0)
    norm = _eyes(sd, S["ids"])
    eyes = C.byref(norm) if eyes_on else None
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
    frames = _frames(sd, S, host, idx, stage_half)
    rc = lib.sd_train_level(ctx.h, None, C.byref(frames), ptr(x0), ptr(xg), n, P // 2, C.c_int64(n), eyes, C.byref(p), C.byref(norm), None,
                            C.c_int64(0), C.byref(reg), 0, ptr(buf), C.c_int64(ld), chunk_rows, ptr(X), ptr(nxt), C.byref(lam))
    assert rc == 0, lib.sd_last_error(ctx.h).decode()
    ctx.sync()
    return X.cpu().numpy(), lam.value, nxt.cpu().numpy()


def _apply(sd, S, hp, X, host, chunk_rows, stage_half=0, eyes_on=True, rows=None):
    import torch
    ctx, lib, ptr = S["ctx"], sd._capi.lib(), sd._capi.ptr
    x0 = torch.from_numpy(S["x0"][slice(None) if rows is None else rows]).cuda()
    idx = torch.from_numpy(S["frames"]).cuda() if rows is None else None
    n, P = x0.shape
    p = sd.HoGParam(*hp)
    D = lib.sd_hog_feature_length(P // 2, C.byref(p))
    ld = (D + 3) // 4 * 4
    buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
    Xd = torch.from_numpy(X).cuda()
    nxt = torch.full((n, P), 7.0, device="cuda")
    norm = _eyes(sd, S["ids"])
    eyes = C.byref(norm) if eyes_on else None
    frames = _frames(sd, S, host, idx, stage_half)
    rc = lib.sd_apply_level(ctx.h, C.byref(frames), ptr(x0), n, P // 2, eyes, C.byref(p), C.byref(norm), None, C.c_int64(0), ptr(Xd),
                            ptr(buf), C.c_int64(ld), chunk_rows, ptr(nxt))
    assert rc == 0, lib.sd_last_error(ctx.h).decode()
    ctx.sync()
    return nxt.cpu().numpy()


def _largest_grey():
    return max(h * _round16(w) for w, h, _ in SPECS)


@pytest.mark.parametrize("hp", [ADAPTIVE, FIXED], ids=["adaptive", "fixed"])
@pytest.mark.parametrize("chunk", ["one", "several"])
@pytest.mark.parametrize("stage", ["roomy", "tight"])
def test_host_route_level_is_the_device_level(sd, setup, hp, chunk, stage):
    S = setup
    n = S["x0"].shape[0]
    rows = n if chunk == "one" else 29
    stage_half = (32 << 20) if stage == "roomy" else _largest_grey()          # tight: a batch holds about one frame's regions
    eyes_on = hp is ADAPTIVE
    gathered = sd._capi.lib().sd_gathered_bytes(S["ctx"].h)
    want = _train(sd, S, hp, False, rows, eyes_on=eyes_on)
    got = _train(sd, S, hp, True, rows, stage_half, eyes_on=eyes_on)
    assert sd._capi.lib().sd_gathered_bytes(S["ctx"].h) > gathered
    assert np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])
    # the sample outside its frame moved like every other (its HOG rows are the zero rows the device route gives)
    assert np.isfinite(got[2]).all()
    a_want = _apply(sd, S, hp, want[0], False, rows, eyes_on=eyes_on)
    a_got = _apply(sd, S, hp, want[0], True, rows, stage_half, eyes_on=eyes_on)
    assert np.array_equal(a_got, a_want)


def test_host_level_without_an_index_reads_frame_i(sd, setup):
    """d_sample_frame NULL on the host route: sample i reads frame i, as with the identity index"""
    S = setup
    first = [int(np.flatnonzero(S["frames"] == f)[0]) for f in range(S["nf"])]   # one sample of each frame, in frame order
    want = _train(sd, S, ADAPTIVE, False, len(first), rows=first)
    got = _train(sd, S, ADAPTIVE, True, len(first), rows=first)
    assert np.array_equal(got[0], want[0]) and got[1] == want[1] and np.array_equal(got[2], want[2])
    assert np.array_equal(_apply(sd, S, ADAPTIVE, want[0], True, 4, rows=first), _apply(sd, S, ADAPTIVE, want[0], False, 4, rows=first))


def test_bad_frames_are_refused_before_any_work(sd, setup):
    import torch
    S = setup
    ctx, lib, ptr = S["ctx"], sd._capi.lib(), sd._capi.ptr
    x0, xg = torch.from_numpy(S["x0"]).cuda(), torch.from_numpy(S["x_gt"]).cuda()
    idx = torch.from_numpy(S["frames"]).cuda()
    n, P = x0.shape
    p = sd.HoGParam(*ADAPTIVE)
    D = lib.sd_hog_feature_length(P // 2, C.byref(p))
    ld = (D + P + 3) // 4 * 4
    buf = torch.empty((n, ld), dtype=torch.float32, device="cuda")
    X = torch.full((D, P), 7.0, device="cuda")
    nxt = torch.full((n, P), 7.0, device="cuda")
    norm = _eyes(sd, S["ids"])
    reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()

    def calls(frames):
        t = lib.sd_train_level(ctx.h, None, C.byref(frames), ptr(x0), ptr(xg), n, P // 2, C.c_int64(n), C.byref(norm), C.byref(p),
                               C.byref(norm), None, C.c_int64(0), C.byref(reg), 0, ptr(buf), C.c_int64(ld), n, ptr(X), ptr(nxt), None)
        a = lib.sd_apply_level(ctx.h, C.byref(frames), ptr(x0), n, P // 2, C.byref(norm), C.byref(p), C.byref(norm), None, C.c_int64(0),
                               ptr(X), ptr(buf), C.c_int64(D + 3 & ~3), n, ptr(nxt))
        return t, a

    recs = [S["table"][i] for i in range(S["nf"])]
    unpinned = np.zeros((97, 144), dtype=np.uint8)                         # pageable, 16-byte pitch
    bad_pin = list(recs)
    bad_pin[2] = sd._host_frame(unpinned[:, :131])[0]
    bad_stride = list(recs)
    r = recs[0]
    bad_stride[0] = sd.HostFrameC(r.h_data, r.width - 8, r.height, r.row_stride - 8, r.channels)   # pitch 152: not a multiple of 16
    launches = ctx.launches()
    for table in (bad_pin, bad_stride):
        assert calls(_frames(sd, S, True, idx, table=(sd.HostFrameC * len(table))(*table))) == (1, 1)
    both = _frames(sd, S, True, idx)
    both.images = C.pointer(S["ib"])
    assert calls(both) == (1, 1) and calls(sd.LevelFramesC(d_sample_frame=ptr(idx))) == (1, 1)   # exactly one source of frames
    assert ctx.launches() == launches
    ctx.sync()
    assert bool((X == 7.0).all()) and bool((nxt == 7.0).all())
    # an index out of range is the projection's status flag, reported by the next synchronising call
    idx[5] = 99
    assert calls(_frames(sd, S, True, idx)) == (0, 0)
    with pytest.raises(sd.SdError) as e:
        ctx.sync()
    assert e.value.code == 1 and "out of range" in str(e.value)


def _python_setup(sd, golden, copies):
    m = sd.load_detection_model(golden.model_path)
    imgs = [synth.smooth_images(1, 120, 160, seed=20 + i)[0] for i in range(24)]
    rng = np.random.default_rng(9)
    frames, x0, x_gt = [], [], []
    for f in range(len(imgs)):
        for k in range(11):
            box = (22 + int(rng.integers(-3, 4)), 8 + int(rng.integers(-3, 4)), 100, 100)
            x_gt.append(sd.align_mean(m.get_mean(), box))
            x0.append(sd.align_mean(m.get_mean(), box, 1 + rng.normal(0, 0.03), 1 + rng.normal(0, 0.03), rng.normal(0, 0.03), rng.normal(0, 0.03)))
            frames.append(imgs[f] if not copies else imgs[f].copy())
    return m.landmark_ids, frames, np.asarray(x0, np.float32), np.asarray(x_gt, np.float32), imgs


def _python_run(sd, ids, frames, x0, x_gt, rows=None):
    hps = [sd.HoGParam(*ADAPTIVE), sd.HoGParam(1, 3, 6, 4, 0.5)]
    ht = sd.HogTransform(frames, hps, ids, REYE, LEYE)
    regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)) for _ in hps]
    sdo = sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(ids, REYE, LEYE))
    xt = sdo.train(x_gt, x0, None, ht, rows_per_chunk=rows).cpu().numpy()
    xs = sdo.test(x0, None, ht, rows_per_chunk=rows).cpu().numpy()
    return ht, [r.x.cpu().numpy() for r in regs] + [xt, xs]


def test_python_shared_frames(sd, golden, monkeypatch):
    ids, shared, x0, x_gt, imgs = _python_setup(sd, golden, copies=False)
    _, copies, _, _, _ = _python_setup(sd, golden, copies=True)
    ht1, one = _python_run(sd, ids, shared, x0, x_gt)
    ht11, eleven = _python_run(sd, ids, copies, x0, x_gt)
    assert ht1.on_device() and ht11.on_device()
    assert ht1.images.numel() == len(imgs) * 120 * 160 and ht11.images.numel() == 11 * len(imgs) * 120 * 160
    assert all(np.array_equal(a, b) for a, b in zip(one, eleven))
    # the same set through image_index: one entry per photo
    ht = sd.HogTransform(imgs, [sd.HoGParam(*ADAPTIVE)], ids, REYE, LEYE, image_index=np.repeat(np.arange(len(imgs)), 11))
    assert np.array_equal(ht(x0, 0).cpu().numpy(), ht1(x0, 0).cpu().numpy())
    # frames that stay in host memory: bit for bit the device route, also through chunks
    monkeypatch.setattr(sd, "DEVICE_FRAME_SHARE", 0.0)
    monkeypatch.setattr(sd, "HOST_STAGE_HALF", 64 << 10)
    hth, host = _python_run(sd, ids, shared, x0, x_gt)
    assert not hth.on_device() and hth.images is None
    assert all(np.array_equal(a, b) for a, b in zip(one, host))
    _, host_chunks = _python_run(sd, ids, shared, x0, x_gt, rows=100)
    monkeypatch.setattr(sd, "DEVICE_FRAME_SHARE", 0.5)
    _, dev_chunks = _python_run(sd, ids, shared, x0, x_gt, rows=100)
    assert all(np.array_equal(a, b) for a, b in zip(dev_chunks, host_chunks))

"""Cascade levels on mirrored samples (SD_SAMPLE_MIRRORED in sd_level_frames.d_sample_frame) against the same levels on a
materialised set: the frames plus np.fliplr copies passed as frames of their own.  X, lambda and x_next must be bit for bit equal,
on the device route and on the host route (grey and colour pinned frames), in one chunk and in several, with the rank diagnostic
on.  The host route must gather no more bytes for a set of samples plus their mirrors than for the materialised set, and
HogTransform(mirrored=...) must hold each frame once and train, test and predict bit for bit as on copies."""
import ctypes as C

import numpy as np
import pytest

import synth

pytestmark = pytest.mark.gpu

BIT = 1 << 30
ADAPTIVE = (1, 3, 8, 4, 1.0)
FIXED = (1, 3, 8, 4, 0.0)         # hog_eyes NULL
REYE, LEYE = ["37", "40"], ["43", "46"]
SPECS = [(160, 120, 1), (201, 150, 3), (131, 97, 1), (176, 144, 3), (97, 96, 1)]     # (w, h, channels); odd widths
PER_FRAME = 6


def _round16(v):
    return (v + 15) // 16 * 16


def _pinned_frame(img):
    """a pinned copy of (h, w) or (h, w, 3) uint8 with a 16-byte aligned base and row pitch, and its array view"""
    import torch
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else 3
    pitch = ch * _round16(w)
    t = torch.empty(h * pitch + 16, dtype=torch.uint8).pin_memory()
    off = (-t.data_ptr()) % 16
    a = t[off:off + h * pitch].numpy().reshape(h, pitch)
    a[:, :w * ch] = img.reshape(h, w * ch)
    return t, np.lib.stride_tricks.as_strided(a, img.shape, (pitch, ch, 1) if ch == 3 else (pitch, 1))


def _images():
    out = []
    for i, (w, h, ch) in enumerate(SPECS):
        g = synth.smooth_images(ch, h, w, seed=40 + i)
        out.append(g[0] if ch == 1 else np.ascontiguousarray(np.moveaxis(g, 0, -1)))
    return out


def _samples(sd, mean, seed=9):
    """PER_FRAME samples of every frame, some over a border, in shuffled order: (frame, x0, x_gt)"""
    rng = np.random.default_rng(seed)
    frame, x0, x_gt = [], [], []
    for f, (w, h, _) in enumerate(SPECS):
        s = min(w, h) * 3 // 4
        for k in range(PER_FRAME):
            over = k % 3 == 2
            bx = int(rng.integers(-s // 3, w - s + s // 3)) if over else (w - s) // 2 + int(rng.integers(-4, 5))
            by = int(rng.integers(-s // 3, h - s + s // 3)) if over else (h - s) // 2 + int(rng.integers(-4, 5))
            x_gt.append(sd.align_mean(mean, (bx, by, s, s)))
            x0.append(sd.align_mean(mean, (bx, by, s, s), 1 + rng.normal(0, 0.04), 1 + rng.normal(0, 0.04), rng.normal(0, 0.04),
                                    rng.normal(0, 0.04)))
            frame.append(f)
    order = rng.permutation(len(frame))
    return np.asarray(frame, dtype=np.int32)[order], np.asarray(x0, dtype=np.float32)[order], np.asarray(x_gt, dtype=np.float32)[order]


class _Set:
    """frames on both routes: the pinned host table and the same frames uploaded by sd_upload_frames"""

    def __init__(self, sd, ctx, imgs):
        import torch
        self.pinned = [_pinned_frame(i) for i in imgs]
        recs = [sd._host_frame(v)[0] for _, v in self.pinned]
        self.table = (sd.HostFrameC * len(recs))(*recs)
        self.n = len(recs)
        lib = sd._capi.lib()
        nbytes = C.c_size_t(0)
        assert lib.sd_upload_frames(ctx.h, self.table, self.n, None, C.byref(nbytes), None) == 0
        self.dbuf = torch.empty(nbytes.value, dtype=torch.uint8, device="cuda")
        self.ib = sd.ImageBatchC()
        assert lib.sd_upload_frames(ctx.h, self.table, self.n, sd._capi.ptr(self.dbuf), C.byref(nbytes), C.byref(self.ib)) == 0

    def frames(self, sd, host, idx):
        f = sd.LevelFramesC(d_sample_frame=sd._capi.ptr(idx), stage_half_bytes=0)
        if host:
            f.host_frames, f.num_host_frames = self.table, self.n
        else:
            f.images = C.pointer(self.ib)
        return f


@pytest.fixture(scope="module")
def setup(sd, golden):
    ctx = sd.default_context()
    m = sd.load_detection_model(golden.model_path, ctx)
    ids = m.landmark_ids
    perm = sd.mirror_permutation(ids)
    imgs = _images()
    mirrors = [np.ascontiguousarray(np.fliplr(i)) for i in imgs]
    frame, x0, x_gt = _samples(sd, m.get_mean())
    width = np.array([w for w, _, _ in SPECS])[frame]
    F = len(imgs)
    # the samples, then their mirrors: in place (the frame index with the bit) and materialised (frame F + f)
    X0 = np.concatenate([x0, sd.mirror_landmarks(x0, width, perm)])
    XG = np.concatenate([x_gt, sd.mirror_landmarks(x_gt, width, perm)])
    idx_in_place = np.concatenate([frame, frame | BIT]).astype(np.int32)
    idx_copies = np.concatenate([frame, frame + F]).astype(np.int32)
    return dict(ctx=ctx, ids=ids, perm=perm, imgs=imgs, mirrors=mirrors, X0=X0, XG=XG, idx_in_place=idx_in_place,
                idx_copies=idx_copies, own=_Set(sd, ctx, imgs), copies=_Set(sd, ctx, imgs + mirrors))


def _level(sd, S, which, hp, host, chunk_rows, train, X=None, idx=None, x0=None):
    """one sd_train_level (X None) or sd_apply_level on the set `which` ("own": the frames, mirrored in place; "copies")"""
    import torch
    ctx, lib, ptr = S["ctx"], sd._capi.lib(), sd._capi.ptr
    x0 = torch.from_numpy(S["X0"] if x0 is None else x0).cuda()
    xg = torch.from_numpy(S["XG"]).cuda()
    idx = torch.from_numpy(S["idx_in_place"] if which == "own" else S["idx_copies"]).cuda() if idx is None else idx
    n, P = x0.shape
    p = sd.HoGParam(*hp)
    D = lib.sd_hog_feature_length(P // 2, C.byref(p))
    norm = sd.InterEyeDistanceNormalisation(S["ids"], REYE, LEYE).c()
    eyes = C.byref(norm) if hp[4] > 0 else None
    frames = S[which].frames(sd, host, idx)
    nxt = torch.full((n, P), 7.0, device="cuda")
    if train:
        ld = (D + P + 3) // 4 * 4
        buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
        Xo = torch.full((D, P), 7.0, device="cuda")
        lam = C.c_float(0)
        reg = sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False).c()
        rc = lib.sd_train_level(ctx.h, None, C.byref(frames), ptr(x0), ptr(xg), n, P // 2, C.c_int64(n), eyes, C.byref(p), C.byref(norm),
                                None, C.c_int64(0), C.byref(reg), 0, ptr(buf), C.c_int64(ld), chunk_rows, ptr(Xo), ptr(nxt), C.byref(lam))
        assert rc == 0, lib.sd_last_error(ctx.h).decode()
        ctx.sync()
        return Xo.cpu().numpy(), lam.value, nxt.cpu().numpy(), ctx.last_rank()
    ld = (D + 3) // 4 * 4
    buf = torch.empty((chunk_rows, ld), dtype=torch.float32, device="cuda")
    Xd = torch.from_numpy(X).cuda()
    rc = lib.sd_apply_level(ctx.h, C.byref(frames), ptr(x0), n, P // 2, eyes, C.byref(p), C.byref(norm), None, C.c_int64(0), ptr(Xd),
                            ptr(buf), C.c_int64(ld), chunk_rows, ptr(nxt))
    assert rc == 0, lib.sd_last_error(ctx.h).decode()
    ctx.sync()
    return nxt.cpu().numpy()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("host", [False, True], ids=["device", "host"])
@pytest.mark.parametrize("chunk", ["one", "several"])
@pytest.mark.parametrize("hp", [ADAPTIVE, FIXED], ids=["adaptive", "fixed"])
def test_mirrored_levels_equal_materialised_levels(sd, setup, host, chunk, hp):
    S = setup
    n = len(S["X0"])
    rows = n if chunk == "one" else 7
    lib = sd._capi.lib()
    S["ctx"].set_rank_diagnostic(chunk == "several")
    try:
        g0 = lib.sd_gathered_bytes(S["ctx"].h)
        got = _level(sd, S, "own", hp, host, rows, True)
        g1 = lib.sd_gathered_bytes(S["ctx"].h)
        want = _level(sd, S, "copies", hp, host, rows, True)
        g2 = lib.sd_gathered_bytes(S["ctx"].h)
    finally:
        S["ctx"].set_rank_diagnostic(False)
    assert np.array_equal(_bits(got[0]), _bits(want[0])), "X"
    assert _bits(got[1]) == _bits(want[1]), "lambda"
    assert np.array_equal(_bits(got[2]), _bits(want[2])), "x_next"
    assert got[3] == want[3], "rank"
    if chunk == "several":
        assert got[3] > 0
    if host:
        print(f"gathered bytes: mirrored in place {g1 - g0}, materialised {g2 - g1}")
        assert 0 < g1 - g0 <= g2 - g1
    apply_got = _level(sd, S, "own", hp, host, rows, False, X=got[0])
    apply_want = _level(sd, S, "copies", hp, host, rows, False, X=got[0])
    assert np.array_equal(_bits(apply_got), _bits(apply_want)), "apply x_next"


def test_mirrored_host_index_out_of_range_flags_the_level(sd, setup):
    """A flagged index past the frame count on the host route raises the status flag, as an unflagged one does."""
    import torch
    S = setup
    idx = torch.from_numpy(S["idx_in_place"].copy()).cuda()
    idx[3] = len(S["imgs"]) | BIT
    with pytest.raises(sd.SdError, match="out of range"):
        _level(sd, S, "own", ADAPTIVE, True, len(S["X0"]), True, idx=idx)
    S["ctx"].sync()


def _optimiser(sd, ids, levels):
    regs = [sd.LinearRegressor(sd.Regulariser(sd.RegularisationType.MatrixNorm, 1.5, False)) for _ in range(levels)]
    return sd.SupervisedDescentOptimiser(regs, sd.InterEyeDistanceNormalisation(ids, REYE, LEYE))


@pytest.mark.parametrize("route", ["device", "host"])
def test_python_mirrored_transform_equals_copies(sd, setup, monkeypatch, route):
    """train / test / predict through HogTransform(mirrored=...) against a transform over the frames and their mirrors, with
    callbacks; the in-place transform holds each frame once."""
    S = setup
    ids, imgs, F = S["ids"], S["imgs"], len(S["imgs"])
    frame = S["idx_in_place"] & ~BIT
    flags = (S["idx_in_place"] & BIT) != 0
    hps = [sd.HoGParam(*ADAPTIVE), sd.HoGParam(1, 3, 6, 4, 0.8)]
    if route == "host":
        monkeypatch.setattr(sd, "DEVICE_FRAME_SHARE", 0.0)
        monkeypatch.setattr(sd, "HOST_STAGE_HALF", 64 << 10)
    own = sd.HogTransform(imgs, hps, ids, REYE, LEYE, image_index=frame, mirrored=flags)
    copies = sd.HogTransform(imgs + S["mirrors"], hps, ids, REYE, LEYE, image_index=S["idx_copies"])
    assert own.on_device() == (route == "device") and copies.on_device() == (route == "device")
    if route == "device":
        assert own.batch().count == F and copies.batch().count == 2 * F
    else:
        assert len(own._host[0]) == F and len(copies._host[0]) == 2 * F
    res = []
    for h in (own, copies):
        sdo = _optimiser(sd, ids, len(hps))
        seen = []
        xt = sdo.train(S["XG"], S["X0"], None, h, on_training_epoch_callback=lambda x: seen.append(x.cpu().numpy()), rows_per_chunk=13)
        xs = sdo.test(S["X0"], None, h, on_regressor_iteration_callback=lambda x: seen.append(x.cpu().numpy()))
        xp = sdo.predict(S["X0"], None, h)
        res.append([r.x.cpu().numpy() for r in sdo.regressors] + [xt.cpu().numpy(), xs.cpu().numpy(), xp.cpu().numpy()] + seen)
    assert len(res[0]) == len(res[1])
    for k, (a, b) in enumerate(zip(*res)):
        assert np.array_equal(_bits(a), _bits(b)), k
    if route == "device":
        # rows through __call__ / debug honour the flags; an explicit training_index reads unmirrored
        x = S["X0"]
        assert np.array_equal(_bits(own(x, 0).cpu().numpy()), _bits(copies(x, 0).cpu().numpy()))
        for a, b in zip(own.debug(x, 1), copies.debug(x, 1)):
            assert np.array_equal(a.cpu().numpy(), b.cpu().numpy())
        t = np.arange(len(x)) % F
        assert np.array_equal(_bits(own(x, 0, training_index=t).cpu().numpy()), _bits(copies(x, 0, training_index=t).cpu().numpy()))


def test_python_mirrored_needs_one_flag_per_sample(sd, setup):
    S = setup
    with pytest.raises(ValueError):
        sd.HogTransform(S["imgs"], [sd.HoGParam(*ADAPTIVE)], S["ids"], REYE, LEYE, image_index=[0, 1, 2], mirrored=[True, False])

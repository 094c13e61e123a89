"""Aligned face chips on the device (sd_face_chips, face_chips, face_chip_template) against the restatement of
tests/face_chip_ref.py, which the CPU tests pin to cv2.warpAffine: chips, both transforms and valid are bit for bit its
  - for grey, B,G,R and float frames, in equally sized, per-frame-size, planar, interleaved and strided batches;
  - for faces taken straight from a track_and_detect step, on the device;
  - for invalid rows (a NaN landmark, all used landmarks equal) mixed with valid ones, which stay unaffected;
  - past 65,535 faces at a small chip size;
and refused calls write nothing, and two runs are identical."""
import ctypes as C

import numpy as np
import pytest
import torch

import face_chip_ref as ref
import synth

pytestmark = pytest.mark.gpu

L = 68


def _frames(C_, dtype, n, H, W, seed):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        g = np.stack([synth.smooth_images(1, H, W, seed=seed + 17 * i + c, sigma=1.0)[0] for c in range(C_)], axis=-1)
        g = g ^ rng.integers(0, 8, g.shape, dtype=np.uint8)
        g = g[:, :, 0] if C_ == 1 else g
        out.append((g.astype(np.float32) / np.float32(255)) if dtype == np.float32 else g)
    return out


def _faces(golden, sizes, per_frame, seed):
    """(face_frame, landmarks (N, 2L) float32): align_mean of random boxes, rotated about the box centre by up to 180 degrees."""
    rng = np.random.default_rng(seed)
    mean = golden.mean68.astype(np.float32).ravel()
    ff, xs = [], []
    for f, (H, W) in enumerate(sizes):
        for _ in range(per_frame):
            s = int(rng.integers(12, max(13, min(H, W))))
            bx, by = int(rng.integers(-s // 3, W - s // 2)), int(rng.integers(-s // 3, H - s // 2))
            x = np.concatenate([(mean[:L] + np.float32(0.5)) * np.float32(s) + np.float32(bx),
                                (mean[L:] + np.float32(0.5)) * np.float32(s) + np.float32(by)]).astype(np.float64)
            t = rng.uniform(-np.pi, np.pi)
            cx, cy = bx + s / 2, by + s / 2
            dx, dy = x[:L] - cx, x[L:] - cy
            xs.append(np.concatenate([cx + np.cos(t) * dx - np.sin(t) * dy, cy + np.sin(t) * dx + np.cos(t) * dy]).astype(np.float32))
            ff.append(f)
    return np.asarray(ff, np.int32), np.stack(xs)


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype == np.uint8 else a.view(np.uint32 if a.dtype == np.float32 else np.uint64)


def _check(got, want):
    g = [t.cpu().numpy() for t in got]
    chips, c2f, f2c, valid = want
    assert g[0].shape == chips.shape and g[0].dtype == chips.dtype
    assert np.array_equal(_bits(g[0]), _bits(chips))
    assert np.array_equal(_bits(g[1]), _bits(c2f.reshape(-1, 2, 3))) and np.array_equal(_bits(g[2]), _bits(f2c.reshape(-1, 2, 3)))
    assert np.array_equal(g[3], valid)


@pytest.mark.parametrize("kind", ["grey", "bgr", "float1", "float3"])
def test_layouts_equal_the_rule(sd, golden, kind):
    C_, dtype = {"grey": (1, np.uint8), "bgr": (3, np.uint8), "float1": (1, np.float32), "float3": (3, np.float32)}[kind]
    size, idx = (40, 48), np.array([36, 39, 42, 45, 30, 48, 54])          # eyes' corners, nose tip, mouth corners
    tm = ref.template(golden.mean68, *size, 0.3, idx)
    frames = _frames(C_, dtype, 3, 90, 120, seed=C_)
    ff, x = _faces(golden, [(90, 120)] * 3, 5, seed=4)
    want = ref.face_chips(frames, ff, x, idx, tm, *size)
    assert want[3].all()
    batch = torch.from_numpy(np.stack(frames)).cuda()
    # equally sized, interleaved (channels last)
    _check(sd.face_chips(batch, ff, x, size, tm, idx, channels_last=True), want)
    # device tensors for face_frame and landmarks
    _check(sd.face_chips(batch, torch.from_numpy(ff).cuda(), torch.from_numpy(x).cuda(), size, tm, idx, channels_last=True), want)
    # planar (count, C, H, W)
    planar = (batch[:, None] if C_ == 1 else batch.permute(0, 3, 1, 2)).contiguous()
    _check(sd.face_chips(planar, ff, x, size, tm, idx), want)
    # strided: every other column of frames twice as wide
    wide = torch.zeros((3, 90, 240) + ((C_,) if C_ > 1 else ()), dtype=batch.dtype, device="cuda")
    wide[:, :, ::2] = batch
    _check(sd.face_chips(wide[:, :, ::2], ff, x, size, tm, idx, channels_last=True), want)
    # per-frame sizes (a list of frames of different sizes)
    mixed = [frames[0], frames[1][:70, :101], frames[2][5:, 7:]]
    mixed = [np.ascontiguousarray(f) for f in mixed]
    ffm, xm = _faces(golden, [f.shape[:2] for f in mixed], 4, seed=5)
    _check(sd.face_chips(mixed, ffm, xm, size, tm, idx, channels_last=True), ref.face_chips(mixed, ffm, xm, idx, tm, *size))


def test_default_template_and_all_landmarks(sd, golden):
    m = sd.load_detection_model(golden.model_path)
    Lm = m.num_landmarks
    tm = sd.face_chip_template(m, 112)
    assert np.array_equal(tm, ref.template(m.get_mean(), 112, 112, 0.25))
    assert np.array_equal(sd.face_chip_template(m, (40, 30), 0.1, [3, 1]), ref.template(m.get_mean(), 40, 30, 0.1, [3, 1]))
    frames = _frames(3, np.uint8, 2, 100, 140, seed=8)
    rng = np.random.default_rng(1)
    x = (m.get_mean().astype(np.float32).reshape(1, -1) * np.float32(60) + np.float32(40)
         + rng.normal(0, 2, (6, 2 * Lm)).astype(np.float32)).astype(np.float32)
    ff = np.array([0, 1, 0, 1, 1, 0], np.int32)
    _check(sd.face_chips(frames, ff, x, 112, tm, channels_last=True), ref.face_chips(frames, ff, x, np.arange(Lm), tm, 112, 112))


def test_faces_from_a_tracking_step(sd, golden):
    """face_frame and landmarks straight out of track_and_detect (CUDA tensors) make the rule's chips."""
    m = sd.load_detection_model(golden.model_path)
    grey = [golden.examples[f"gray{i}"] for i in range(5)]
    K, FW, FH = 9, 6, 6
    rng = np.random.default_rng(3)
    filt = torch.from_numpy(rng.normal(0, 0.1, (3 * K + 4, FH, FW)).astype(np.float32)).cuda()
    scales = [2.0 ** (-k / 4) for k in range(2, 14)]
    neg = float("-inf")
    r = m.track_and_detect(grey, [], np.zeros((0, 2 * m.num_landmarks), np.float32), (filt, 0.0), (FW, FH), 8, K, neg, scales,
                           range(5), neg, max_detections=3)
    assert r.num_new > 0 and r.frame.is_cuda and r.landmarks.is_cuda
    tm = sd.face_chip_template(m, (64, 80))
    got = sd.face_chips(grey, r.frame, r.landmarks, (64, 80), tm)
    want = ref.face_chips(grey, r.frame.cpu().numpy(), r.landmarks.cpu().numpy(), np.arange(m.num_landmarks), tm, 64, 80)
    _check(got, want)


def test_invalid_rows_leave_the_others_alone(sd, golden):
    size, idx = (32, 32), np.arange(L)
    tm = ref.template(golden.mean68, *size, 0.25)
    frames = _frames(3, np.uint8, 2, 80, 100, seed=11)
    ff, x = _faces(golden, [(80, 100)] * 2, 4, seed=12)
    bad = x.copy()
    bad[1, 5] = np.nan                                 # a NaN used landmark
    bad[4, :L], bad[4, L:] = 20.0, 30.0                # every used landmark equal
    bad[6] *= np.float32(1e30)                         # a fixed-point coordinate leaves int32
    want = ref.face_chips(frames, ff, bad, idx, tm, *size)
    assert want[3].tolist() == [True, False, True, True, False, True, False, True]
    _check(sd.face_chips(frames, ff, bad, size, tm, idx, channels_last=True), want)
    good = sd.face_chips(frames, ff, x, size, tm, idx, channels_last=True)
    got = sd.face_chips(frames, ff, bad, size, tm, idx, channels_last=True)
    keep = torch.tensor(want[3], device="cuda")
    assert torch.equal(got.chips[keep], good.chips[keep]) and torch.equal(got.chip_to_frame[keep], good.chip_to_frame[keep])


def test_past_65535_faces(sd, golden):
    frames = _frames(1, np.float32, 4, 60, 70, seed=21)
    ff, x = _faces(golden, [(60, 70)] * 4, 40, seed=22)
    reps = 70000 // len(ff) + 1
    ffb, xb = np.tile(ff, reps)[:70000], np.tile(x, (reps, 1))[:70000]
    idx = np.array([36, 45, 30, 48, 54])
    tm = ref.template(golden.mean68, 5, 4, 0.2, idx)
    got = sd.face_chips(frames, ffb, xb, (5, 4), tm, idx, channels_last=True)
    head = ref.face_chips(frames, ff, x, idx, tm, 5, 4)
    g = [t.cpu().numpy() for t in got]
    for i, t in enumerate(g):
        w = np.asarray(head[i])
        tiled = np.tile(w, (reps,) + (1,) * (w.ndim - 1))[:70000]
        assert np.array_equal(_bits(t), _bits(tiled.reshape(t.shape)))


def test_two_runs_are_identical(sd, golden):
    frames = torch.from_numpy(np.stack(_frames(3, np.float32, 2, 64, 64, seed=31))).cuda()
    ff, x = _faces(golden, [(64, 64)] * 2, 30, seed=32)
    tm = ref.template(golden.mean68, 48, 48, 0.25)
    a = sd.face_chips(frames, ff, x, 48, tm, channels_last=True)
    b = sd.face_chips(frames, ff, x, 48, tm, channels_last=True)
    for s, t in zip(a, b):
        assert torch.equal(s.view(torch.uint8) if s.dtype != torch.bool else s, t.view(torch.uint8) if t.dtype != torch.bool else t)


def test_refusals_write_nothing(sd, golden):
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    lib = _capi.lib()
    frames = torch.from_numpy(np.stack(_frames(3, np.uint8, 2, 50, 60, seed=41))).cuda()
    _, ib, _ = sd._hog_images(frames, True, ctx, lambda w, h: None)
    ff, x = _faces(golden, [(50, 60)] * 2, 3, seed=42)
    n = len(ff)
    dff, dx = torch.from_numpy(ff).cuda(), torch.from_numpy(x).cuda()
    chips = torch.full((n, 16, 16, 3), 77, dtype=torch.uint8, device="cuda")
    c2f = torch.full((n, 6), 7.0, dtype=torch.float64, device="cuda")
    f2c = torch.full((n, 6), 7.0, dtype=torch.float64, device="cuda")
    valid = torch.full((n,), 9, dtype=torch.uint8, device="cuda")

    def call(face=dff, idx=np.arange(L), w=16, h=16, nl=L, ldl=2 * L, tmpl=None, images=ib):
        idx = np.ascontiguousarray(idx, np.int32)
        tm = np.ascontiguousarray(ref.template(golden.mean68, max(w, 1), max(h, 1), 0.25, idx % L) if tmpl is None else tmpl)
        p = _capi.FaceChipParamC(w, h, idx.size, idx.ctypes.data_as(C.c_void_p), tm.ctypes.data_as(C.c_void_p))
        return lib.sd_face_chips(ctx.h, C.byref(images), _capi.ptr(face), _capi.ptr(dx), ldl, n, nl, C.byref(p), _capi.ptr(chips),
                                 _capi.ptr(c2f), _capi.ptr(f2c), _capi.ptr(valid))

    def unchanged():
        torch.cuda.synchronize()
        return bool((chips == 77).all() and (c2f == 7).all() and (f2c == 7).all() and (valid == 9).all())

    bad_frame = torch.tensor(ff, device="cuda")
    bad_frame[2] = 2                                                   # frame index out of range (checked on the device)
    assert call(face=bad_frame) == 1 and unchanged()
    bad_frame[2] = -1
    assert call(face=bad_frame) == 1 and unchanged()
    assert call(idx=[36, 45, 36]) == 1 and unchanged()                 # an index listed twice
    assert call(idx=[36, 68]) == 1 and unchanged()                     # an index out of range
    assert call(idx=[36]) == 1 and unchanged()                         # n < 2
    assert call(w=0) == 1 and unchanged()                              # a chip below 1 x 1
    assert call(h=-3) == 1 and unchanged()
    assert call(ldl=2 * L - 1) == 1 and unchanged()
    neg = _capi.HogImagesC.from_buffer_copy(ib)
    neg.frame.row_stride = -1                                          # a negative stride
    assert call(images=neg) == 1 and unchanged()
    four = _capi.HogImagesC.from_buffer_copy(ib)
    four.channels = 17
    assert call(images=four) == 1 and unchanged()
    # the context still works: a good call after the refusals
    assert call() == 0
    torch.cuda.synchronize()
    assert (valid == 1).all()

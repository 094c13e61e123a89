"""The landmark HOG kernel's word-wide pixel stages (hog_patch_kernel, csrc/sd_hog.cu): the resize that writes two output
columns per thread from word loads of the staged window, and the gradient pass that takes runs of four pixels, against the
oracle's restatement of cv::resize and of hog.c's orientation bins, at every compiled-in schedule (K = 4 and 9, fs = 55 /
50 / 40 / 30).

Faces: bench.py's frames and boxes at a seed of their own.  Each face's landmarks are scaled about the face centre by a
factor from 0.45 to 2.4, so the windows span at least three TMA box classes at every cell size (all eight
over the four), and every fourth face is moved over a frame edge or
corner.  The same frames are also laid out with an odd row stride, which stages every window by byte loads; both layouts
must give the oracle's patches and bins, byte for byte.
"""
import ctypes as C

import numpy as np
import pytest

N = 64
SEED = 97
SCHEDULES = [(K, cs) for K in (4, 9) for cs in (11, 10, 8, 6)]


@pytest.fixture(scope="module")
def faces(sd):
    """(context, model, frames on the host, landmark rows (N, 2L), eye normalisation, {layout: (image batch, kept tensor)})."""
    import torch
    import bench
    from superviseddescent_b200 import _capi
    ctx = sd.Context(0)
    model = sd.load_detection_model(bench.MODEL, ctx)
    frames = bench.synth_frames_numpy(N, SEED)
    boxes = bench.synth_boxes(N, SEED)
    L = model.num_landmarks
    rng = np.random.default_rng(SEED)
    x = np.stack([sd.align_mean(model.get_mean(), b) for b in boxes]).astype(np.float64)
    W, H = bench.W_IMG, bench.H_IMG
    for i in range(N):
        xs, ys = x[i, :L], x[i, L:]
        mx, my = xs.mean(), ys.mean()
        s = 0.45 + (2.4 - 0.45) * i / (N - 1)
        xs[:] = mx + s * (xs - mx)
        ys[:] = my + s * (ys - my)
        if i % 4 == 1:                                       # over an edge or a corner
            tx = (-mx + 10.0, W - mx - 10.0, 0.0)[i % 3]
            ty = (0.0, -my + 5.0, H - my - 5.0)[(i // 3) % 3]
            xs += tx
            ys += ty
    x += rng.normal(0.0, 1.5, x.shape)
    x = x.astype(np.float32)
    norm = sd.NormalisationC()
    _capi.lib().sd_model_normalisation(model._m, C.byref(norm))
    dense = torch.from_numpy(frames).cuda()
    odd = torch.zeros((N, H, W + 1), dtype=torch.uint8, device="cuda")
    odd[:, :, :W] = dense
    layouts = {
        "frames": (sd.ImageBatchC(C.c_void_p(dense.data_ptr()), W, H, dense.stride(1), dense.stride(0), N), dense),
        "odd-stride": (sd.ImageBatchC(C.c_void_p(odd.data_ptr()), W, H, odd.stride(1), odd.stride(0), N), odd),
    }
    return ctx, model, frames, x, norm, layouts


def _param(model, K, cs):
    for level in range(model.num_levels):
        hp = model.hog_param(level)
        if hp.cell_size == cs:
            hp.num_bins = K
            return hp
    raise AssertionError(f"the shipped model has no level with cell size {cs}")


@pytest.mark.gpu
@pytest.mark.parametrize("K,cs", SCHEDULES, ids=[f"K{K}-cs{cs}" for K, cs in SCHEDULES])
def test_patches_and_bins_equal_the_oracle(sd, oracle, faces, K, cs):
    import torch
    from superviseddescent_b200 import _capi
    ctx, model, frames, x, norm, layouts = faces
    lib = _capi.lib()
    L = model.num_landmarks
    hp = _param(model, K, cs)
    fs = hp.num_cells * cs
    xd = torch.from_numpy(x).cuda()
    got = {}
    for name, (ib, _) in layouts.items():
        geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
        patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
        bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
        rc = lib.sd_hog_debug(ctx.h, C.byref(ib), None, _capi.ptr(xd), C.c_int64(xd.stride(0)), N, L, C.byref(norm), C.byref(hp),
                              _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
        assert rc == 0, lib.sd_last_error(ctx.h)
        assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
        got[name] = (geo.cpu().numpy(), patches.cpu().numpy(), bins.cpu().numpy())
    geo = got["frames"][0]
    assert np.array_equal(got["odd-stride"][0], geo)
    P = 2 * geo[:, :, 2]
    boxes = (32, 48, 64, 80, 96, 112, 128, 160)
    reached = {min((b for b in boxes if b >= p), default=None) for p in P.ravel()}
    assert len(reached - {None}) >= 3, f"windows of {P.min()}-{P.max()} px reach the box classes {sorted(b for b in reached if b)}"
    cx, cy, half = geo[:, :, 0], geo[:, :, 1], geo[:, :, 2]
    H, W = frames.shape[1:]
    assert np.any(cx - half < 0) and np.any(cy - half < 0) and np.any(cx + half > W) and np.any(cy + half > H)
    want_p = np.empty((N, L, fs, fs), np.uint8)
    want_b = np.empty((N, L, fs, fs), np.int32)
    for i in range(N):
        for l in range(L):
            q = oracle.resize_linear_u8(oracle.crop_patch_u8(frames[i], int(cx[i, l]), int(cy[i, l]), int(half[i, l])), fs, fs)
            want_p[i, l] = q
            want_b[i, l] = oracle.hog_orientation_bins(q.astype(np.float32), K)
    for name, (_, patches, bins) in got.items():
        bad = np.any(patches != want_p, axis=(2, 3))
        assert not bad.any(), f"{name}, K={K} cs={cs}: patches of {int(bad.sum())} windows differ from cv::resize (P = {sorted(set(P[bad].tolist()))[:8]})"
        bad = np.any(bins.astype(np.int32) != want_b, axis=(2, 3))
        assert not bad.any(), f"{name}, K={K} cs={cs}: bins of {int(bad.sum())} windows differ from hog.c"

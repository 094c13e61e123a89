"""The landmark HOG kernel's compiled-in schedules (hog_patch_kernel<K, 5, cs, T>, csrc/sd_hog.cu), each at the CTA size that
launch_hog picks for it: K = 4 and 9, cell sizes 11 / 10 / 8 / 6 (fs = 55 / 50 / 40 / 30).

Faces: bench.py's frames and boxes at a seed of their own, the shipped model's mean shape aligned to each box and jittered by
a few pixels, so the eye-normalised windows differ in size from face to face and some reach over the frame's edge.  N = 233
faces of L = 22 landmarks: N * L = 5126 patches, a multiple of no CTA size and of no patches-per-CTA count of the
normalisation kernel.

  - Every landmark row equals, bit for bit, the dense HOG (sd_hog_dense, a separate kernel) of the resized fs x fs patches
    that sd_hog_debug returns for the same faces.  This takes the eye-normalised route with resizing, since the fixed-patch
    route needs an even cell size and cannot reach cs = 11.
  - Every face's row is bit-identical whether the face is computed alone, in a batch of 7 or in the batch of all N.
"""
import ctypes as C

import numpy as np
import pytest

N = 233
SEED = 4321
SCHEDULES = [(K, cs) for K in (4, 9) for cs in (11, 10, 8, 6)]
SINGLES = list(range(0, N, 19)) + [N - 1]


@pytest.fixture(scope="module")
def faces(sd):
    """(context, model, image batch, kept tensors, landmark rows (N, 2L) on the device, eye normalisation)."""
    import torch
    import bench
    from superviseddescent_b200 import _capi
    ctx = sd.Context(0)
    model = sd.load_detection_model(bench.MODEL, ctx)
    frames = torch.from_numpy(bench.synth_frames_numpy(N, SEED)).cuda()
    boxes = bench.synth_boxes(N, SEED)
    rng = np.random.default_rng(SEED)
    x = np.stack([sd.align_mean(model.get_mean(), b) for b in boxes]).astype(np.float32)
    x += rng.normal(0.0, 3.0, x.shape).astype(np.float32)
    norm = sd.NormalisationC()
    _capi.lib().sd_model_normalisation(model._m, C.byref(norm))
    ib = sd.ImageBatchC(C.c_void_p(frames.data_ptr()), bench.W_IMG, bench.H_IMG, frames.stride(1), frames.stride(0), N)
    return ctx, model, ib, frames, torch.from_numpy(x).cuda(), norm


def _param(model, K, cs):
    """The model level's HOG parameters (variant, cells, relative patch size) at this cell size and bin count."""
    for level in range(model.num_levels):
        hp = model.hog_param(level)
        if hp.cell_size == cs:
            hp.num_bins = K
            return hp
    raise AssertionError(f"the shipped model has no level with cell size {cs}")


def _rows(faces, hp, first, count):
    """sd_hog_batch of faces [first, first + count) as one batch: (count, D) float32 on the host."""
    import torch
    from superviseddescent_b200 import _capi
    ctx, model, ib, _, x, norm = faces
    lib = _capi.lib()
    L = model.num_landmarks
    D = lib.sd_hog_feature_length(L, C.byref(hp))
    idx = torch.arange(first, first + count, dtype=torch.int32, device="cuda")
    A = torch.full((count, D), float("nan"), dtype=torch.float32, device="cuda")
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x[first:first + count]), C.c_int64(x.stride(0)), count,
                          L, C.byref(norm), C.byref(hp), _capi.ptr(A), C.c_int64(D))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    return A.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("K,cs", SCHEDULES, ids=[f"K{K}-cs{cs}" for K, cs in SCHEDULES])
def test_landmark_rows_equal_dense_hog_of_their_patches(sd, faces, K, cs):
    import torch
    from superviseddescent_b200 import _capi
    ctx, model, ib, _, x, norm = faces
    lib = _capi.lib()
    L, nc = model.num_landmarks, 5
    hp = _param(model, K, cs)
    assert hp.num_cells == nc
    fs = nc * cs
    geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
    patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
    bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
    rc = lib.sd_hog_debug(ctx.h, C.byref(ib), None, _capi.ptr(x), C.c_int64(x.stride(0)), N, L, C.byref(norm), C.byref(hp),
                          _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    half = geo[:, :, 2].cpu().numpy()
    assert len(np.unique(half)) > 3, "the windows should differ in size from face to face"
    assert np.any(2 * half != fs), "the windows should be resized"
    rows = _rows(faces, hp, 0, N)
    dd = 3 * K + 4 if hp.variant == 1 else 4 * K
    dense = sd.hog_dense(patches.reshape(N * L, fs, fs), cs, K, hp.variant, ctx=ctx).cpu().numpy()
    assert dense.shape == (N * L, dd, nc, nc)
    want = dense.reshape(N, L, dd, nc, nc).transpose(0, 1, 2, 4, 3).reshape(N, L * dd * nc * nc)   # per-dimension transpose
    got = rows[:, :-1]
    same = np.all(got.view(np.uint32) == want.view(np.uint32), axis=1)
    assert same.all(), f"K={K} cs={cs}: rows of faces {np.flatnonzero(~same).tolist()[:8]} differ from the dense HOG of their patches"
    assert np.all(rows[:, -1] == 1.0)


@pytest.mark.gpu
@pytest.mark.parametrize("K,cs", SCHEDULES, ids=[f"K{K}-cs{cs}" for K, cs in SCHEDULES])
def test_rows_do_not_depend_on_the_batch(sd, faces, K, cs):
    model = faces[1]
    hp = _param(model, K, cs)
    whole = _rows(faces, hp, 0, N).view(np.uint32)
    sevens = np.concatenate([_rows(faces, hp, b, min(7, N - b)) for b in range(0, N, 7)]).view(np.uint32)
    same = np.all(sevens == whole, axis=1)
    assert same.all(), f"K={K} cs={cs}: faces {np.flatnonzero(~same).tolist()[:8]} differ between batches of 7 and of {N}"
    for i in SINGLES:
        one = _rows(faces, hp, i, 1).view(np.uint32)
        assert np.array_equal(one[0], whole[i]), f"K={K} cs={cs}: face {i} alone differs from face {i} in the batch of {N}"

"""The HOG kernel's orientation bin against the reference expression (hog.c:645-672, the oracle's hog_orientation_bins) for
EVERY integer gradient an 8-bit patch can have, (gx, gy) in [-255, 255]^2, at every bin count K in 1..16.

The kernel decides most bins without a division, by a margin test on the un-normalised gradient, and evaluates the
reference expression only where that margin is too small; a wrong margin or a wrong fallback shows up here as a pixel
whose bin differs.  Each frame is the fixed (un-resized) 54 x 54 patch of FixedHogTransform (9 cells of 6 px), laid out
as 3 x 3 crosses at stride 3, so that the centre pixel of every cross gets a gradient chosen freely: left / right and
top / bottom neighbours max(0, -g), max(0, -g) + g.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NC, CS = 9, 6
FS = NC * CS                      # 54: fits the kernel's shared-memory layout at K = 16
CENTRES = np.arange(1, FS - 1, 3)  # 18 per side, all interior


def _frames():
    g = np.arange(-255, 256)
    gx, gy = [v.ravel() for v in np.meshgrid(g, g, indexing="xy")]
    per = CENTRES.size ** 2
    n = -(-gx.size // per)
    pad = n * per - gx.size
    gx = np.concatenate([gx, np.zeros(pad, dtype=gx.dtype)]).reshape(n, CENTRES.size, CENTRES.size)
    gy = np.concatenate([gy, np.zeros(pad, dtype=gy.dtype)]).reshape(n, CENTRES.size, CENTRES.size)
    frames = np.zeros((n, FS, FS), dtype=np.uint8)
    cy, cx = np.meshgrid(CENTRES, CENTRES, indexing="ij")
    left, top = np.maximum(0, -gx), np.maximum(0, -gy)
    f = np.arange(n)[:, None, None]
    frames[f, cy, cx - 1] = left
    frames[f, cy, cx + 1] = left + gx
    frames[f, cy - 1, cx] = top
    frames[f, cy + 1, cx] = top + gy
    return frames, gx, gy


def test_orientation_bin_every_gradient_every_k(sd, oracle):
    import torch
    from superviseddescent_b200 import _capi
    frames, gx, gy = _frames()
    n = frames.shape[0]
    d = frames.astype(np.int32)
    cy, cx = np.meshgrid(CENTRES, CENTRES, indexing="ij")
    assert np.array_equal(d[:, cy, cx + 1] - d[:, cy, cx - 1], gx) and np.array_equal(d[:, cy + 1, cx] - d[:, cy - 1, cx], gy)
    pairs = set(zip(gx.ravel().tolist(), gy.ravel().tolist()))
    assert len(pairs) == 511 * 511                                          # every gradient of an 8-bit patch
    x = torch.full((n, 2), FS / 2, dtype=torch.float32, device="cuda")      # L = 1 landmark at the frame's centre
    for K in range(1, 17):
        h = sd.FixedHogTransform(frames, 0, NC, CS, K)
        ctx = h.ctx
        geo = torch.empty((n, 1, 3), dtype=torch.int32, device="cuda")
        patches = torch.empty((n, 1, FS, FS), dtype=torch.uint8, device="cuda")
        bins = torch.empty((n, 1, FS, FS), dtype=torch.int8, device="cuda")
        rc = _capi.lib().sd_hog_debug(ctx.h, C.byref(h._batch), None, _capi.ptr(x), C.c_int64(x.stride(0)), n, 1, None,
                                      C.byref(h.param), _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
        assert rc == 0, _capi.lib().sd_last_error(ctx.h)
        assert np.array_equal(patches[:, 0].cpu().numpy(), frames), K
        got = bins[:, 0].cpu().numpy().astype(np.int32)
        # one tall image: rows 1..52 and columns 1..52 of every frame see only their own frame's pixels
        ref = oracle.hog_orientation_bins(frames.reshape(n * FS, FS).astype(np.float32), K).reshape(n, FS, FS)
        assert np.array_equal(got[:, 1:-1, 1:-1], ref[:, 1:-1, 1:-1]), \
            f"K={K}: {int(np.sum(got[:, 1:-1, 1:-1] != ref[:, 1:-1, 1:-1]))} interior pixels differ"

"""The orientation bin by sector search (hog_bin in csrc/sd_hog_common.cuh) for every integer gradient an 8-bit image can have,
(gx, gy) in [-255, 255]^2, at every bin count K in 1..16: in the landmark kernel (sd_hog_debug) and in the dense kernel
(sd_hog_dense), against the reference expression (the oracle's hog_orientation_bins); the share of gradients whose margin
test fails and that take the reference expression, counted by a float32 restatement of the margin test on the host (the
kernels do not report which pixels fall back); and the feature rows of the four detect levels on faces from bench.py's host
frames and boxes, bit for bit against the fingerprints in tests/golden/hog_levels_ref.npz (tests/golden/gen_hog_levels.py),
which were made with the build before the sector search.
"""
import ctypes as C
import importlib.util
import math
import os

import numpy as np
import pytest

from test_gpu_hog_orientation import CENTRES, CS, FS, NC, _frames

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _centre_bins(oracle, frames, K):
    """The reference's bin at the centre of every cross of the frames, (n, 18, 18)."""
    n = frames.shape[0]
    ref = oracle.hog_orientation_bins(frames.reshape(n * FS, FS).astype(np.float32), K).reshape(n, FS, FS)
    cy, cx = np.meshgrid(CENTRES, CENTRES, indexing="ij")
    return ref[:, cy, cx]


def _sector_fast_path(gx, gy, K):
    """The sector search's accepted bins, restated in float32 on the host: (bins, accepted).  fmaf(b, y, -p) is the double sum
    b * y + p rounded once to float, which is exact because b * y and p span fewer than 53 bits."""
    bx = np.array([np.float32(math.cos((2 * j + 1) * math.pi / (2 * K))) for j in range(K // 2)], dtype=np.float32)
    by = np.array([np.float32(math.sin((2 * j + 1) * math.pi / (2 * K))) for j in range(K // 2)], dtype=np.float32)
    margin = np.float32(4e-6 / (2.0 * math.sin(math.pi / (2 * K))))
    fx, fy = np.abs(gx).astype(np.float32), np.abs(gy).astype(np.float32)
    g = np.sqrt((gx * gx + gy * gy).astype(np.float32))
    m = fx.copy() if K % 2 else np.full(fx.shape, np.inf, dtype=np.float32)
    s = np.zeros(fx.shape, dtype=np.int64)
    for j in range(K // 2):
        p = (by[j] * fx).astype(np.float32)
        c = (np.float64(bx[j]) * fy.astype(np.float64) - p.astype(np.float64)).astype(np.float32)
        s += c > 0
        m = np.minimum(m, np.abs(c))
    accepted = m > (margin * g).astype(np.float32)
    neg = gy < 0
    s = np.where((gx < 0) != neg, K - s, s) + np.where(neg, K, 0)
    return np.where(s < 2 * K, s, 0), accepted


def test_sector_margin_on_the_host(oracle):
    """Where the host restatement of the margin test accepts, the sector is the reference's bin; the rest (nearly all exactly
    on a sector boundary) take the reference expression, and their share is printed.  The restatement builds the boundary
    directions and the margin with the same libm expressions as hog_orientations and rounds every operation as hog_bin does."""
    frames, gx, gy = _frames()
    for K in range(1, 17):
        bins, accepted = _sector_fast_path(gx.astype(np.int64), gy.astype(np.int64), K)
        ref = _centre_bins(oracle, frames, K)
        assert np.array_equal(bins[accepted], ref[accepted]), f"K={K}: {int(np.sum(bins[accepted] != ref[accepted]))} bins differ"
        real = ~accepted & (gx != 0)                       # gx = 0 takes the axis rule, g = 0 is bin -1: no reference expression
        frac = float(real.sum()) / (511 * 511)
        print(f"K={K:2d}: {int(real.sum())} of 261121 gradients take the reference expression ({100 * frac:.4f} %)")
        assert frac < 0.005, K


@pytest.mark.gpu
def test_sector_bins_every_gradient_landmark_and_dense(sd, oracle):
    """Every gradient at every K: the landmark kernel's bins against the reference, and the dense kernel's features of the same
    frames against the landmark kernel's, bit for bit (the dense HOG of an fs x fs frame is the fixed-patch row)."""
    import torch
    from superviseddescent_b200 import _capi
    frames, gx, gy = _frames()
    n = frames.shape[0]
    x = torch.full((n, 2), FS / 2, dtype=torch.float32, device="cuda")
    dframes = torch.from_numpy(frames).cuda()
    for K in range(1, 17):
        h = sd.FixedHogTransform(frames, 1, NC, CS, K)
        geo = torch.empty((n, 1, 3), dtype=torch.int32, device="cuda")
        patches = torch.empty((n, 1, FS, FS), dtype=torch.uint8, device="cuda")
        bins = torch.empty((n, 1, FS, FS), dtype=torch.int8, device="cuda")
        rc = _capi.lib().sd_hog_debug(h.ctx.h, C.byref(h._batch), None, _capi.ptr(x), C.c_int64(x.stride(0)), n, 1, None,
                                      C.byref(h.param), _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
        assert rc == 0, _capi.lib().sd_last_error(h.ctx.h)
        cy, cx = np.meshgrid(CENTRES, CENTRES, indexing="ij")
        got = bins[:, 0].cpu().numpy().astype(np.int32)[:, cy, cx]
        ref = _centre_bins(oracle, frames, K)
        assert np.array_equal(got, ref), f"K={K}: {int(np.sum(got != ref))} gradients differ"
        row = h(x.cpu().numpy(), 0).cpu().numpy()
        dd = 3 * K + 4
        dense = sd.hog_dense(dframes, CS, K, 1).cpu().numpy()
        assert dense.shape == (n, dd, NC, NC)
        assert np.array_equal(dense.transpose(0, 1, 3, 2).reshape(n, -1), row[:, :dd * NC * NC]), K


@pytest.mark.gpu
def test_detect_level_rows_match_the_committed_fingerprints():
    """The feature rows of levels 0..3 on 64 bench-seeded faces, bit for bit against the fingerprints of the build before the
    sector search."""
    spec = importlib.util.spec_from_file_location("gen_hog_levels", os.path.join(GOLDEN, "gen_hog_levels.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    want = np.load(os.path.join(GOLDEN, "hog_levels_ref.npz"))
    rows = gen.level_rows()
    for level, r in rows.items():
        same = np.all(gen.fingerprints(r) == want[f"sha256_{level}"], axis=1)
        assert same.all(), (f"level {level}: rows {np.flatnonzero(~same).tolist()} differ; sums "
                            f"{r.astype(np.float64).sum(axis=1)[~same][:4]} against {want[f'sum_{level}'][~same][:4]}")

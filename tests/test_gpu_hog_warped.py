"""Warped samples in the landmark HOG kernel (sd_hog_batch_warped / sd_hog_debug_warped) against the unwarped calls on the
materialised virtual frames (cv2.warpAffine(..., WARP_INVERSE_MAP) of each sample's frame, passed as a frame of its own), bit for
bit: geometry, resized patches, orientation bins and feature rows.

The samples are test_gpu_hog_configs.py's route cases (windows at every staged size, the next, unstaged one, across every border
and wholly outside), read in V's coordinates, so both window routes of the WARP kernel run at every compiled-in schedule and at the
run-time K = 4 and K = 9 ones.  Each sample of one frame gets its own warp (rotations, scales, reflections, shear, V smaller and
larger than the frame) in one launch; the frame-table layout mixes frame sizes.  The identity warp gives the unwarped rows, the
reflection [-1, 0, W - 1; 0, 1, 0] the mirrored route's, and invalid warps, a mirrored bit and d_roi batches are refused."""
import ctypes as C

import numpy as np
import pytest
import torch

import sample_warp_ref as SW
import test_gpu_hog_configs as HC
from superviseddescent_b200 import _capi

pytestmark = pytest.mark.gpu

L = HC.L
BIT = 1 << 30
CONFIGS = [(1, 5, cs, K) for K in (4, 9) for cs in (11, 10, 8, 6)] + [(1, 8, 10, 4), (0, 3, 4, 9)]


def _warp_of(sd, k, W, H):
    """warp k of a frame W x H: (M, (Wv, Hv))"""
    c = (W / 2 + 3.5, H / 2 - 2.25)
    kinds = [
        (sd.rotation_warp(c, 0.0), (W, H)),
        (sd.rotation_warp(c, 37.0), (W, H)),
        (sd.rotation_warp(c, -90.0, 0.5), (W + 40, max(H - 30, 8))),
        (sd.rotation_warp(c, 180.0, 2.0), (W // 2, H // 2)),
        (np.array([[-1.0, 0, W - 1], [0, 1, 0]]), (W, H)),
        (np.array([[0.8, 0.35, -7.3], [-0.15, 1.3, 4.1]]), (W, H)),
        (sd.rotation_warp(c, -21.5, 1.4), (W + 3, H + 5)),
    ]
    return kinds[k % len(kinds)]


def _table(warps):
    rec = np.zeros(len(warps), dtype=[("m", "<f8", (6,)), ("w", "<i4"), ("h", "<i4")])
    for i, (M, (w, h)) in enumerate(warps):
        rec[i] = (np.asarray(M, np.float64).ravel(), w, h)
    return torch.from_numpy(rec.view(np.uint8).copy()).cuda()


def _run(ctx, ib, samples, cfg, warps=None):
    """(geometry, patches, bins, feature bits) of sd_hog_debug[_warped] and sd_hog_batch[_warped]"""
    lib = _capi.lib()
    fs = cfg[1] * cfg[2]
    N = len(samples)
    x = torch.from_numpy(np.stack([r for _, r in samples])).cuda()
    idx = torch.tensor([f for f, _ in samples], dtype=torch.int32, device="cuda")
    p = HC._param(cfg)
    eyes = HC._eyes()
    geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
    patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
    bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.full((N, D), float("nan"), dtype=torch.float32, device="cuda")
    head = (ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, C.byref(eyes), C.byref(p))
    if warps is None:
        rc = lib.sd_hog_debug(*head, _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
        assert rc == 0, lib.sd_last_error(ctx.h)
        rc = lib.sd_hog_batch(*head, _capi.ptr(A), C.c_int64(D))
    else:
        w = _table(warps)
        rc = lib.sd_hog_debug_warped(*head, _capi.ptr(w), _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
        assert rc == 0, lib.sd_last_error(ctx.h)
        rc = lib.sd_hog_batch_warped(*head, _capi.ptr(w), _capi.ptr(A), C.c_int64(D))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    return [geo.cpu().numpy(), patches.cpu().numpy(), bins.cpu().numpy(), A.cpu().numpy().view(np.uint32)]


def _diff(got, want, what):
    names = ("geometry", "patches", "bins", "features")
    return [f"{what}: {n} differ in {int(np.sum(np.any((g != w).reshape(len(g), -1), axis=1)))} samples"
            for n, g, w in zip(names, got, want) if not np.array_equal(g, w)]


def _materialised(frames, samples, warps):
    """one V per sample, as the frame-table layout, and the samples reading V i"""
    vs = [SW.materialise(frames[f], M, size) for (f, _), (M, size) in zip(samples, warps)]
    return HC.Layout("frames", vs), [(i, r) for i, (_, r) in enumerate(samples)]


def test_warped_samples_equal_materialised_frames_on_both_routes(sd):
    ctx = sd.default_context()
    frames = HC._frames()
    bad, table = [], []
    for cfg in CONFIGS:
        assert HC.accepted(cfg), cfg
        common, small = HC.route_samples(cfg)
        cap = HC.smem_layout(cfg)[0]
        for kind in ("tma", "frames"):
            samples = common + (small if kind == "frames" else [])
            lay = HC.Layout(kind, frames)
            warps = [_warp_of(sd, k, lay.frames[f].shape[1], lay.frames[f].shape[0]) for k, (f, _) in enumerate(samples)]
            ib, keep, _ = HC.device_batch(lay)
            got = _run(ctx, ib, samples, cfg, warps)
            lay_v, own = _materialised(lay.frames, samples, warps)
            ib_v, keep_v, _ = HC.device_batch(lay_v)
            want = _run(ctx, ib_v, own, cfg)
            bad += _diff(got, want, f"{cfg} {kind}")
        # both window routes: a staged warped window holds (P + 30 & ~15) x P bytes and 16 P bytes of terms
        Ps = {int(r[1] - r[0]) for _, r in common}
        staged = {P for P in Ps if (((P + 30) & ~15) + 16) * P <= cap}
        assert staged and staged != Ps, (cfg, sorted(Ps))
        table.append(f"{str(cfg):<16} staged P {sorted(staged)[-1]}, unstaged P {sorted(Ps - staged)[0]}")
    print("\n" + "\n".join(table))
    assert not bad, "\n".join(bad[:40])


def test_identity_and_reflection_warps(sd):
    """The identity warp at the frame's size gives the unwarped rows; the reflection gives the mirrored route's rows."""
    ctx = sd.default_context()
    frames = HC._frames()
    for cfg in ((1, 5, 10, 4), (1, 5, 8, 9), (1, 8, 10, 4)):
        common, _ = HC.route_samples(cfg)
        lay = HC.Layout("tma", frames)
        ib, keep, _ = HC.device_batch(lay)
        W = lay.frames[0].shape[1]
        ident = [(np.eye(2, 3), (HC.W, HC.H))] * len(common)
        assert not _diff(_run(ctx, ib, common, cfg, ident), _run(ctx, ib, common, cfg), f"{cfg} identity")
        refl = [(np.array([[-1.0, 0, W - 1], [0, 1, 0]]), (HC.W, HC.H))] * len(common)
        mirrored = [(f | BIT, r) for f, r in common]
        assert not _diff(_run(ctx, ib, common, cfg, refl), _run(ctx, ib, mirrored, cfg), f"{cfg} reflection")


def test_refusals(sd):
    lib = _capi.lib()
    ctx = sd.default_context()
    lay = HC.Layout("tma", HC._frames())
    ib, keep, _ = HC.device_batch(lay)
    cfg = (1, 5, 6, 4)
    p, eyes = HC._param(cfg), HC._eyes()
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.zeros((1, D), dtype=torch.float32, device="cuda")
    x = torch.from_numpy(HC._sample(0, 40, (10, 10), (50, 50))[1][None]).cuda()

    def call(idx, M, size, batch=ib):
        d_idx = torch.tensor([idx], dtype=torch.int32, device="cuda")
        w = _table([(M, size)])
        return lib.sd_hog_batch_warped(ctx.h, C.byref(batch), _capi.ptr(d_idx), _capi.ptr(x), C.c_int64(2 * L), 1, L, C.byref(eyes),
                                       C.byref(p), _capi.ptr(w), _capi.ptr(A), C.c_int64(D))

    for M, size in ((np.array([[np.nan, 0, 0], [0, 1, 0]]), (50, 50)), (np.eye(2, 3), (0, 50)), (np.eye(2, 3), (50, -1)),
                    (np.array([[1e9, 0, 0], [0, 1, 0]]), (50, 50)), (np.array([[1, 0, 3e6], [0, 1, 0]]), (50, 50))):
        assert call(0, M, size) == 0
        assert lib.sd_sync(ctx.h) == 1, (M, size)
        assert "invalid sample warp" in lib.sd_last_error(ctx.h).decode()
        assert lib.sd_sync(ctx.h) == 0
    for idx in (0 | BIT, 2, -1):
        assert call(idx, np.eye(2, 3), (50, 50)) == 0
        assert lib.sd_sync(ctx.h) == 1, idx
        assert "out of range" in lib.sd_last_error(ctx.h).decode()
        assert lib.sd_sync(ctx.h) == 0
    # a d_roi batch and a NULL table are refused before any work
    roi_lay = HC.Layout("roi", HC._frames(), [(0, 0, 64, 64), (0, 0, 64, 64)])
    ib_roi, keep_roi, _ = HC.device_batch(roi_lay)
    launches = ctx.launches()
    assert call(0, np.eye(2, 3), (50, 50), ib_roi) == 1
    d_idx = torch.zeros(1, dtype=torch.int32, device="cuda")
    assert lib.sd_hog_batch_warped(ctx.h, C.byref(ib), _capi.ptr(d_idx), _capi.ptr(x), C.c_int64(2 * L), 1, L, C.byref(eyes), C.byref(p),
                                   None, _capi.ptr(A), C.c_int64(D)) == 1
    assert ctx.launches() == launches
    assert lib.sd_sync(ctx.h) == 0

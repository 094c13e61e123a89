"""Mirrored samples in the landmark HOG kernel (SD_SAMPLE_MIRRORED in sd_hog_batch / sd_hog_debug's image index) against the same
samples on materialised mirrors (np.fliplr of each frame passed as a frame of its own), bit for bit: geometry, resized patches,
orientation bins and feature rows.

A mirrored sample's landmark x' = W - x reads the frame's window [x - half, x + half) right to left, so the windows of
tests/test_gpu_hog_configs.py's route cases, given as mirrored samples, reach the kernel's staging through every route that
file's layouts force (every TMA box class, vec16, words, the byte loop and the unstaged resize), across all four borders and
wholly outside the frame.  Each launch also holds the same windows unmirrored, which must equal a launch of their own.  The
frame-table layout holds an odd-width frame beside two 400 x 320 frames; the ROI layout uploads each frame's window hull, and
its mirror uploads the mirrored hull."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_hog_configs as HC
from superviseddescent_b200 import _capi

pytestmark = pytest.mark.gpu

BIT = 1 << 30
L = HC.L
# every compiled-in schedule (nc = 5, K = 4 and 9), the run-time K = 4 and K = 9 kernels and the generic one
CONFIGS = [(1, 5, cs, K) for K in (4, 9) for cs in (11, 10, 8, 6)] + [(1, 8, 10, 4), (0, 3, 4, 9), (1, 1, 4, 1)]
ODD = (21, 27)                      # (h, w) of the odd-width frame of the frame-table layout


def _frames():
    fr = HC._frames()
    fr[2] = np.random.default_rng(7).integers(0, 256, ODD, dtype=np.uint8)
    return fr


def _mirror_row(row, W):
    """The mirrored sample whose windows are the frame windows of row: x' = W - x (its centre in the mirror's coordinates)."""
    out = row.copy()
    out[:L] = np.float32(W) - row[:L]
    return out


def _run(ctx, ib, samples, cfg, adaptive):
    lib = _capi.lib()
    fs = cfg[1] * cfg[2]
    N = len(samples)
    x = torch.from_numpy(np.stack([r for _, r in samples])).cuda()
    idx = torch.tensor([f for f, _ in samples], dtype=torch.int32, device="cuda")
    p = HC._param(cfg)
    eyes = C.byref(HC._eyes()) if adaptive else None
    geo = torch.empty((N, L, 3), dtype=torch.int32, device="cuda")
    patches = torch.empty((N, L, fs, fs), dtype=torch.uint8, device="cuda")
    bins = torch.empty((N, L, fs, fs), dtype=torch.int8, device="cuda")
    rc = lib.sd_hog_debug(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, eyes, C.byref(p),
                          _capi.ptr(geo), _capi.ptr(patches), _capi.ptr(bins))
    assert rc == 0, lib.sd_last_error(ctx.h)
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.full((N, D), float("nan"), dtype=torch.float32, device="cuda")
    rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(idx), _capi.ptr(x), C.c_int64(2 * L), N, L, eyes, C.byref(p),
                          _capi.ptr(A), C.c_int64(D))
    assert rc == 0, lib.sd_last_error(ctx.h)
    assert lib.sd_sync(ctx.h) == 0, lib.sd_last_error(ctx.h)
    return [geo.cpu().numpy(), patches.cpu().numpy(), bins.cpu().numpy(), A.cpu().numpy().view(np.uint32)]


def _rois(common):
    """The hull of each big frame's windows, clipped to the frame (as test_gpu_hog_configs.route_plan), and its mirror."""
    rois = []
    for f in (0, 1):
        wins = [(x, y, int(r[1] - r[0])) for s, r in common if s == f for x, y in HC._windows_of(r, int(r[1] - r[0]))]
        x0 = max(0, min(x for x, _, _ in wins)); y0 = max(0, min(y for _, y, _ in wins))
        x1 = min(HC.W, max(x + P for x, _, P in wins)); y1 = min(HC.H, max(y + P for _, y, P in wins))
        rois.append((x0, y0, x1 - x0, y1 - y0))
    return rois, [(HC.W - x - w, y, w, h) for x, y, w, h in rois]


def _diff(got, want, what):
    names = ("geometry", "patches", "bins", "features")
    return [f"{what}: {n} differ in {int(np.sum(np.any((g != w).reshape(len(g), -1), axis=1)))} samples"
            for n, g, w in zip(names, got, want) if not np.array_equal(g, w)]


@pytest.mark.parametrize("adaptive", [True, False], ids=["adaptive", "fixed"])
def test_mirrored_samples_equal_materialised_mirrors_on_every_route(sd, adaptive):
    ctx = sd.default_context()
    frames = _frames()
    mirrors = [np.ascontiguousarray(np.fliplr(f)) for f in frames]
    bad, table = [], []
    for cfg in CONFIGS:
        assert HC.accepted(cfg), cfg
        if not adaptive and cfg[2] % 2:
            continue                                          # the fixed transform needs an even cell size
        common, small = HC.route_samples(cfg)
        rois_f, rois_m = _rois(common)
        cap = HC.smem_layout(cfg)[0]
        routes = set()
        for kind in HC.LAYOUTS:
            samples = common + (small if kind == "frames" else [])
            lay_f = HC.Layout(kind, frames, rois_f if kind == "roi" else None)
            lay_m = HC.Layout(kind, mirrors, rois_m if kind == "roi" else None)
            width = [f.shape[1] for f in lay_f.frames]
            mirrored = [(f | BIT, _mirror_row(r, width[f])) for f, r in samples]
            for f, r in samples:
                P = int(r[1] - r[0])
                routes |= {HC.route(cap, P, x0, y0, lay_f.desc[f]) for x0, y0 in HC._windows_of(r, P)}
            ib_f, keep_f, miss_f = HC.device_batch(lay_f)
            ib_m, keep_m, miss_m = HC.device_batch(lay_m)
            got = _run(ctx, ib_f, mirrored + samples, cfg, adaptive)                 # mirrored and unmirrored in one launch
            want_m = _run(ctx, ib_m, [(f & ~BIT, r) for f, r in mirrored], cfg, adaptive)
            want_u = _run(ctx, ib_f, samples, cfg, adaptive)
            n = len(samples)
            bad += _diff([g[:n] for g in got], want_m, f"{cfg} {kind} mirrored")
            bad += _diff([g[n:] for g in got], want_u, f"{cfg} {kind} unmirrored beside mirrored")
            for miss, what in ((miss_f, "frames"), (miss_m, "mirrors")):
                if miss is not None and miss.cpu().numpy().any():
                    bad.append(f"{cfg} roi: d_roi_miss set on the {what} although the ROI covers every window")
        if adaptive:
            assert routes == HC.allowed_routes(cfg), (cfg, routes)
        table.append(f"{str(cfg):<16} {sorted(routes)}")
    print("\n" + "\n".join(table))
    assert not bad, "\n".join(bad[:40])


def test_mirrored_index_out_of_range_flags_the_next_sync(sd):
    """A flagged index past the frame count, and a flagged face_frame in detect, raise "image index out of range"."""
    lib = _capi.lib()
    ctx = sd.default_context()
    ib, keep, _ = HC.device_batch(HC.Layout("tma", HC._frames()))     # two frames
    cfg = (1, 5, 6, 4)
    p, eyes = HC._param(cfg), HC._eyes()
    D = lib.sd_hog_feature_length(L, C.byref(p))
    A = torch.zeros((1, D), dtype=torch.float32, device="cuda")
    x = torch.from_numpy(HC._sample(0, 40, (10, 10), (50, 50))[1][None]).cuda()
    for idx in (2 | BIT, -(1 << 31) | BIT, 2):
        d_idx = torch.tensor([idx], dtype=torch.int32, device="cuda")
        rc = lib.sd_hog_batch(ctx.h, C.byref(ib), _capi.ptr(d_idx), _capi.ptr(x), C.c_int64(2 * L), 1, L, C.byref(eyes),
                              C.byref(p), _capi.ptr(A), C.c_int64(D))
        assert rc == 0, lib.sd_last_error(ctx.h)
        assert lib.sd_sync(ctx.h) == 1, idx
        assert "image index out of range" in lib.sd_last_error(ctx.h).decode()
        assert lib.sd_sync(ctx.h) == 0


def test_detect_treats_the_bit_as_out_of_range(sd, golden):
    """sd_detect_faces_device's face_frame is not a sample map: frame 0 | SD_SAMPLE_MIRRORED is out of range there."""
    import synth
    m = sd.load_detection_model(golden.model_path)
    images = torch.from_numpy(synth.smooth_images(2, 240, 320, seed=3)).cuda()
    box = synth.face_boxes(1, 240, 320, seed=3)[0]
    x0 = torch.from_numpy(sd.align_mean(m.get_mean(), box)[None]).cuda()
    m.detect_batch_device(images, x0, image_index=[1])
    with pytest.raises(sd.SdError, match="out of range"):
        m.detect_batch_device(images, x0, image_index=[BIT])
    sd.default_context().sync()

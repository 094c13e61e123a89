"""The dense HOG pyramid on the device (sd_hog_pyramid, api.vl_hog_pyramid): every non-empty level is bit for bit sd_hog_dense of
oracle.resize_linear_u8(frame, level_w, level_h) (cv2.resize INTER_LINEAR, checked on the CPU in test_hog_pyramid_shape.py),
the scale-1 level is sd_hog_dense of the frame itself, empty levels and the floats around every level are left alone, and
invalid calls are refused before any work."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

CANARY = -12345.5


def _frame(h, w, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 127.5 + 90 * np.sin(x / 13.0 + np.cos(y / 17.0)) * np.cos(y / 9.0) + rng.normal(0, 12, (h, w))
    img = np.clip(np.round(img), 0, 255).astype(np.uint8)
    img[h // 3:h // 3 + max(1, h // 8), :] = 77
    return img


def _level_ref(sd, oracle, frame, lw, lh, cs, K, variant):
    lvl = frame if (lw, lh) == (frame.shape[1], frame.shape[0]) else oracle.resize_linear_u8(frame, lw, lh)
    return sd.hog_dense(torch.from_numpy(np.ascontiguousarray(lvl))[None].cuda(), cs, K, variant)[0]


SCALES = [1.0, 0.5, 1.5, 2 ** -0.2, 2 ** -0.6, 0.37, 2.0, 0.04]


@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (4, 4, 0), (11, 16, 1), (8, 16, 0), (4, 9, 1), (11, 4, 0)])
def test_mixed_sizes_bit_exact(sd, oracle, cs, K, variant):
    frames = [_frame(97, 131, 1), _frame(120, 160, 2), _frame(45, 61, 3), _frame(13, 200, 4)]
    feats, sizes = sd.vl_hog_pyramid(frames, SCALES, cs, K, variant)
    empty = 0
    for f, frame in enumerate(frames):
        for s, scale in enumerate(SCALES):
            lw, lh = sizes[f][s]
            assert (lw, lh) == (math.floor(frame.shape[1] * scale + 0.5), math.floor(frame.shape[0] * scale + 0.5))
            (_, _), (dd, hh, hw) = sd.hog_pyramid_shape(frame.shape[1], frame.shape[0], scale, cs, K, variant)
            if hw == 0:
                assert feats[f][s] is None
                empty += 1
                continue
            ref = _level_ref(sd, oracle, frame, lw, lh, cs, K, variant)
            assert feats[f][s].shape == ref.shape == (dd, hh, hw)
            assert torch.equal(feats[f][s], ref), (f, scale)
    assert empty > 0


@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (4, 16, 0)])
def test_equal_sizes_with_row_stride(sd, oracle, cs, K, variant):
    n, h, w = 3, 90, 117
    frames = np.stack([_frame(h, w, 10 + i) for i in range(n)])
    wide = torch.zeros((n, h, w + 27), dtype=torch.uint8)
    wide[:, :, :w] = torch.from_numpy(frames)
    dev = wide.cuda()[:, :, :w]                                   # row stride w + 27, frame stride h * (w + 27)
    assert dev.stride(1) == w + 27
    feats, sizes = sd.vl_hog_pyramid(dev, [1.0, 0.5, 1.5, 0.8], cs, K, variant)
    for f in range(n):
        assert torch.equal(feats[f][0], sd.hog_dense(torch.from_numpy(frames[f])[None].cuda(), cs, K, variant)[0])
        for s in range(4):
            lw, lh = sizes[f][s]
            assert torch.equal(feats[f][s], _level_ref(sd, oracle, frames[f], lw, lh, cs, K, variant))


def _call(sd, ib, scales, cs, K, variant, out, offsets):
    ctx = sd.default_context()
    h_scales = (C.c_double * max(len(scales), 1))(*scales)
    from superviseddescent_b200 import _capi
    return _capi.lib().sd_hog_pyramid(ctx.h, C.byref(ib), h_scales, len(scales), cs, K, variant,
                                      _capi.ptr(out), _capi.ptr(offsets))


def test_canaries_and_gaps(sd, oracle):
    """Levels written at caller offsets with gaps; empty levels' offsets point at canaries that must stay untouched."""
    from superviseddescent_b200._capi import ImageBatchC
    cs, K, variant = 8, 9, 1
    frames = np.stack([_frame(70, 83, 20 + i) for i in range(2)])
    t = torch.from_numpy(frames).cuda()
    ib = ImageBatchC(C.c_void_p(t.data_ptr()), 83, 70, 83, 70 * 83, 2)
    scales = [1.0, 0.03, 1.3, 0.25]
    offsets, pos, spans = [], 17, []
    for f in range(2):
        for s in scales:
            (lw, lh), (dd, hh, hw) = sd.hog_pyramid_shape(83, 70, s, cs, K, variant)
            offsets.append(pos if hw else 3)                      # an empty level's offset points into the leading canaries
            if hw:
                spans.append((pos, dd * hh * hw, f, lw, lh))
            pos += dd * hh * hw + 29
    out = torch.full((pos + 50,), CANARY, dtype=torch.float32, device="cuda")
    d_off = torch.tensor(offsets, dtype=torch.int64, device="cuda")
    assert _call(sd, ib, scales, cs, K, variant, out, d_off) == 0
    torch.cuda.synchronize()
    mask = torch.ones_like(out, dtype=torch.bool)
    for p, n, f, lw, lh in spans:
        ref = _level_ref(sd, oracle, frames[f], lw, lh, cs, K, variant)
        assert torch.equal(out[p:p + n], ref.reshape(-1))
        mask[p:p + n] = False
    assert bool((out[mask] == CANARY).all())
    assert len(spans) == 6


def test_refusals_leave_output_untouched(sd):
    from superviseddescent_b200._capi import ImageBatchC
    t = torch.zeros((1, 40, 40), dtype=torch.uint8, device="cuda")
    out = torch.full((10000,), CANARY, dtype=torch.float32, device="cuda")
    off = torch.zeros(4, dtype=torch.int64, device="cuda")
    ib = ImageBatchC(C.c_void_p(t.data_ptr()), 40, 40, 40, 1600, 1)
    for scales, cs, K, variant in [([5.0], 8, 9, 1), ([float("nan")], 8, 9, 1), ([float("inf")], 8, 9, 1), ([0.0], 8, 9, 1),
                                   ([1.0, -1.0], 8, 9, 1), ([], 8, 9, 1), ([1.0], 0, 9, 1), ([1.0], 8, 17, 1), ([1.0], 8, 9, 3)]:
        assert _call(sd, ib, scales, cs, K, variant, out, off) == 1, (scales, cs, K, variant)
    roi = torch.zeros(8, dtype=torch.int32, device="cuda")
    ib.d_roi = C.c_void_p(roi.data_ptr())
    assert _call(sd, ib, [1.0], 8, 9, 1, out, off) == 1
    torch.cuda.synchronize()
    assert bool((out == CANARY).all())

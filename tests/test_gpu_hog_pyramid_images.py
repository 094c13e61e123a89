"""The colour HOG pyramid on the device (sd_hog_pyramid_images, api.vl_hog_pyramid(multichannel=True)).

Every non-empty level is bit for bit sd_hog_dense_images (vl_hog) of oracle.resize_linear_u8 applied to each channel, with the
same channels and orientation mode; one channel with nearest bins is sd_hog_pyramid; three identical channels are one channel;
planar, interleaved and strided views agree; a frame's levels do not depend on its batch or on the scratch slices; the floats
around every level are left alone; the features are within hog.c's 1e-4 bar on cv2-resized colour levels; and invalid calls
are refused before anything is written."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import synth
from conftest import rel_err

pytestmark = pytest.mark.gpu

CANARY = -12345.5
SCALES = [1.0, 0.5, 2.0, 2 ** -0.6, 0.37, 0.04]


def _frame(h, w, c, seed):
    planes = [synth.smooth_images(1, h, w, seed=seed + 11 * k, sigma=1.0)[0] for k in range(c)]
    return np.ascontiguousarray(np.stack(planes, -1))


def _resize(oracle, frame, lw, lh):
    if (lw, lh) == (frame.shape[1], frame.shape[0]):
        return frame
    return np.stack([oracle.resize_linear_u8(frame[..., k], lw, lh) for k in range(frame.shape[2])], -1)


def _bits(t):
    return t.contiguous().view(torch.int32)


def _equal(a, b):
    assert len(a) == len(b)
    for fa, fb in zip(a, b):
        assert len(fa) == len(fb)
        for x, y in zip(fa, fb):
            assert (x is None) == (y is None)
            if x is not None:
                assert x.shape == y.shape and torch.equal(_bits(x), _bits(y))


def _raw(sd, data, frame, image_stride, count, channels, scales, cs, K, variant, bil, dtype=0, frames=None):
    """sd_hog_pyramid_images through the C ABI -> (rc, output buffer with a canary around every level, [(offset, size)])."""
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    ib = _capi.HogImagesC()
    ib.d_data, ib.dtype, ib.channels, ib.count = data.data_ptr(), dtype, channels, count
    ib.frame = _capi.HogImageC(*frame)
    ib.image_stride = image_stride
    ib.d_frames = frames.data_ptr() if frames is not None else None
    w, h = frame[0], frame[1]
    offs, pos = [], 7
    for _ in range(count):
        for s in scales:
            (_, _), (dd, hh, hw) = sd.hog_pyramid_shape(w, h, s, cs, K, variant)
            offs.append((pos, dd * hh * hw))
            pos += dd * hh * hw + 5
    out = torch.full((pos + 7,), CANARY, dtype=torch.float32, device="cuda")
    d_off = torch.tensor([o for o, _ in offs], dtype=torch.int64, device="cuda")
    sc = (C.c_double * len(scales))(*scales)
    rc = _capi.lib().sd_hog_pyramid_images(ctx.h, C.byref(ib), sc, len(scales), cs, K, variant, int(bil), C.c_void_p(out.data_ptr()),
                                           C.c_void_p(d_off.data_ptr()))
    torch.cuda.synchronize()
    return rc, out, offs


@pytest.mark.parametrize("c", [1, 3, 4, 16])
@pytest.mark.parametrize("bil", [False, True])
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("cs,K", [(8, 9), (4, 4), (11, 16)])
def test_levels_are_dense_images_of_the_per_channel_resize(sd, oracle, c, bil, variant, cs, K):
    frames = [_frame(97, 131, c, 1), _frame(45, 61, c, 2), _frame(13, 200, c, 3)]
    feats, sizes = sd.vl_hog_pyramid(frames, SCALES, cs, K, variant, multichannel=True, bilinear_orientations=bil)
    levels, where, empty = [], [], 0
    for f, frame in enumerate(frames):
        for s, scale in enumerate(SCALES):
            lw, lh = sizes[f][s]
            assert (lw, lh) == (math.floor(frame.shape[1] * scale + 0.5), math.floor(frame.shape[0] * scale + 0.5))
            (_, _), (dd, hh, hw) = sd.hog_pyramid_shape(frame.shape[1], frame.shape[0], scale, cs, K, variant)
            if hw == 0:
                assert feats[f][s] is None
                empty += 1
                continue
            levels.append(_resize(oracle, frame, lw, lh))
            where.append((f, s, (dd, hh, hw)))
    assert empty > 0
    ref = sd.vl_hog(levels, cs, K, variant, bilinear_orientations=bil, channels_last=True)
    for (f, s, shape), r in zip(where, ref):
        assert tuple(feats[f][s].shape) == shape == tuple(r.shape)
        assert torch.equal(_bits(feats[f][s]), _bits(r)), (f, SCALES[s])


@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (4, 16, 0)])
def test_one_channel_nearest_is_the_grey_pyramid(sd, cs, K, variant):
    grey = [_frame(97, 131, 1, 5)[..., 0], _frame(120, 160, 1, 6)[..., 0], _frame(45, 61, 1, 7)[..., 0]]
    want, wsizes = sd.vl_hog_pyramid(grey, SCALES, cs, K, variant)
    got, gsizes = sd.vl_hog_pyramid(grey, SCALES, cs, K, variant, multichannel=True)     # a descriptor table: hog_images_kernel
    assert gsizes == wsizes
    _equal(got, want)
    same = np.stack([grey[1]] * 3)
    batch = torch.from_numpy(same).cuda()
    _equal(sd.vl_hog_pyramid(batch, SCALES, cs, K, variant, multichannel=True)[0], sd.vl_hog_pyramid(batch, SCALES, cs, K, variant)[0])
    hwc = torch.from_numpy(same[..., None]).cuda()                                         # pixel stride 1, (count, H, W, 1)
    _equal(sd.vl_hog_pyramid(hwc, SCALES, cs, K, variant, multichannel=True)[0], sd.vl_hog_pyramid(batch, SCALES, cs, K, variant)[0])


@pytest.mark.parametrize("bil", [False, True])
def test_identical_channels_are_one_channel(sd, bil):
    grey = [_frame(97, 131, 1, 8)[..., 0], _frame(64, 80, 1, 9)[..., 0]]
    three = [np.ascontiguousarray(np.stack([g] * 3, -1)) for g in grey]
    one = sd.vl_hog_pyramid(grey, SCALES, 8, 9, 1, multichannel=True, bilinear_orientations=bil)[0]
    _equal(sd.vl_hog_pyramid(three, SCALES, 8, 9, 1, multichannel=True, bilinear_orientations=bil)[0], one)


@pytest.mark.parametrize("bil", [False, True])
def test_planar_interleaved_and_strided_views_agree(sd, bil):
    n, h, w, c, cs, K, v = 3, 90, 117, 3, 8, 9, 1
    frames = np.stack([_frame(h, w, c, 20 + i) for i in range(n)])
    want = sd.vl_hog_pyramid(torch.from_numpy(frames).cuda(), SCALES, cs, K, v, multichannel=True, bilinear_orientations=bil)[0]
    # strided: rows wider than the pixels and a fourth channel that is not read, read in place
    wide = torch.zeros((n, h, w + 21, c + 1), dtype=torch.uint8)
    wide[:, :, :w, :c] = torch.from_numpy(frames)
    wide[:, :, :, c] = 255
    _equal(sd.vl_hog_pyramid(wide.cuda()[:, :, :w, :c], SCALES, cs, K, v, multichannel=True, bilinear_orientations=bil)[0], want)
    _equal(sd.vl_hog_pyramid(list(frames), SCALES, cs, K, v, multichannel=True, bilinear_orientations=bil)[0], want)
    # planar (C, H, W) per frame through the C ABI: pixel stride 1, channel stride H * W
    planar = torch.from_numpy(np.ascontiguousarray(frames.transpose(0, 3, 1, 2))).cuda()
    rc, out, offs = _raw(sd, planar, (w, h, 0, w, 1, h * w), c * h * w, n, c, SCALES, cs, K, v, bil)
    assert rc == 0
    flat = [t for row in want for t in row]
    for (o, size), t in zip(offs, flat):
        if t is None:
            assert size == 0
        else:
            assert torch.equal(_bits(out[o:o + size]), _bits(t.reshape(-1)))
        assert (out[o - 5:o] == CANARY).all() and (out[o + size:o + size + 5] == CANARY).all()


def test_frames_are_batch_independent(sd):
    frames = [_frame(97, 131, 3, 30), _frame(120, 160, 3, 31), _frame(45, 61, 3, 32), _frame(13, 200, 3, 33)]
    for bil in (False, True):
        together = sd.vl_hog_pyramid(frames, SCALES, 8, 9, 1, multichannel=True, bilinear_orientations=bil)[0]
        for f, frame in enumerate(frames):
            _equal([together[f]], sd.vl_hog_pyramid([frame], SCALES, 8, 9, 1, multichannel=True, bilinear_orientations=bil)[0])
        rev = sd.vl_hog_pyramid(frames[::-1], SCALES, 8, 9, 1, multichannel=True, bilinear_orientations=bil)[0]
        _equal(rev[::-1], together)


def test_batch_over_several_scratch_slices(sd):
    # 640 x 480 x 3 at scale 4 is 14.7 MB of levels: six frames need two 64 MB slices, and the frames differ in size
    frames = [_frame(480 - 8 * i, 640 - 12 * i, 3, 40 + i) for i in range(6)]
    scales = [4.0, 1.0, 0.5]
    ctx = sd.default_context()
    before = ctx.launches()
    together = sd.vl_hog_pyramid(frames, scales, 8, 9, 1, multichannel=True)[0]
    torch.cuda.synchronize()
    launches = ctx.launches() - before
    assert launches >= 4, launches                              # a resize and a HOG launch per slice
    for f, frame in enumerate(frames):
        _equal([together[f]], sd.vl_hog_pyramid([frame], scales, 8, 9, 1, multichannel=True)[0])


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_ref
    vl_hog_ref.build()
    if not vl_hog_ref.available():
        pytest.fail("oracle/_ref (the reference's hog.c with channels) is not built: run build()")
    return vl_hog_ref


@pytest.mark.parametrize("bil", [False, True])
def test_levels_within_hog_c_bar_on_cv2_levels(sd, ref, bil):
    cv2 = pytest.importorskip("cv2")
    frame = _frame(120, 160, 3, 50)
    worst = 0.0
    for cs, K, variant in [(8, 9, 1), (4, 4, 0), (11, 16, 1)]:
        feats, sizes = sd.vl_hog_pyramid([frame], SCALES, cs, K, variant, multichannel=True, bilinear_orientations=bil)
        for s in range(len(SCALES)):
            if feats[0][s] is None:
                continue
            lw, lh = sizes[0][s]
            lvl = cv2.resize(frame, (lw, lh), interpolation=cv2.INTER_LINEAR) if (lw, lh) != (160, 120) else frame
            want = ref.vl_hog(np.ascontiguousarray(lvl.transpose(2, 0, 1)).astype(np.float32), cs, K, variant, bil)
            e = rel_err(feats[0][s].cpu().numpy(), want)
            worst = max(worst, e)
            assert e <= 1e-4, (cs, K, variant, SCALES[s], e)
    print(f"colour pyramid against hog.c: worst rel err {worst:.2e}")


def test_refusals_write_nothing(sd):
    from superviseddescent_b200 import _capi
    h, w = 40, 50
    u8 = torch.from_numpy(_frame(h, w, 3, 60)).cuda()
    f32 = u8.float()
    hwc = (w, h, 0, 3 * w, 3, 1)
    cases = [dict(data=f32, dtype=1), dict(channels=0), dict(channels=17), dict(scales=[0.0]), dict(scales=[4.5]),
             dict(scales=[1.0, float("nan")]), dict(frame=(w, h, 0, -3 * w, 3, 1)), dict(frame=(w, h, 0, 3 * w, -3, 1)),
             dict(frame=(w, h, 0, 3 * w, 3, -1)), dict(frame=(w, h, -1, 3 * w, 3, 1)), dict(frame=(0, h, 0, 3 * w, 3, 1)),
             dict(image_stride=-1, count=2), dict(bil=2)]
    ctx = sd.default_context()
    out = torch.empty(1 << 16, dtype=torch.float32, device="cuda")
    for kw in cases:
        a = dict(data=u8, frame=hwc, image_stride=0, count=1, channels=3, scales=[1.0, 0.5], bil=0, dtype=0)
        a.update(kw)
        ib = _capi.HogImagesC()
        ib.d_data, ib.dtype, ib.channels, ib.count = a["data"].data_ptr(), a["dtype"], a["channels"], a["count"]
        ib.frame = _capi.HogImageC(*a["frame"])
        ib.image_stride, ib.d_frames = a["image_stride"], None
        out.fill_(CANARY)
        d_off = torch.zeros(a["count"] * len(a["scales"]), dtype=torch.int64, device="cuda")
        scales = (C.c_double * len(a["scales"]))(*a["scales"])
        rc = _capi.lib().sd_hog_pyramid_images(ctx.h, C.byref(ib), scales, len(a["scales"]), 8, 9, 1, a["bil"],
                                               C.c_void_p(out.data_ptr()), C.c_void_p(d_off.data_ptr()))
        torch.cuda.synchronize()
        print("refused:", kw, _capi.lib().sd_last_error(ctx.h).decode())
        assert rc == 1, kw
        assert (out == CANARY).all(), kw
    with pytest.raises(sd.SdError):
        sd.vl_hog_pyramid(f32, [1.0], 8, 9, 1, multichannel=True)
    with pytest.raises(ValueError):
        sd.vl_hog_pyramid(u8[None], [1.0], 8, 9, 1, bilinear_orientations=True)

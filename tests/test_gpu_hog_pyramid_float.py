"""The float HOG pyramid on the device (sd_hog_pyramid_float, api.vl_hog_pyramid(multichannel=True, float_frames=True)).

Every non-empty level is bit for bit sd_hog_dense_images (vl_hog) of hog_resize_f32_ref.resize_f32, the float rule restated on
the CPU, with the same channels and orientation mode, non-finite and subnormal pixels included; float frames holding integers
give the 8-bit colour pyramid's levels where both rules are exact; planar, interleaved and strided views agree; a frame's levels
do not depend on its batch or on the scratch slices; the floats around every level are left alone; the features are within
hog.c's 1e-4 bar on the restated levels; and invalid calls are refused before anything is written."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import synth
from conftest import rel_err
from hog_resize_f32_ref import resize_f32

pytestmark = pytest.mark.gpu

CANARY = -12345.5
SCALES = [1.0, 0.5, 2.0, 2 ** -0.6, 0.37, 0.04]


def _frame(h, w, c, seed):
    """Smooth float frames with values off the 8-bit grid: a scaled and shifted sum of smooth planes."""
    rng = np.random.default_rng(seed)
    planes = [synth.smooth_images(1, h, w, seed=seed + 11 * k, sigma=1.0)[0].astype(np.float32) for k in range(c)]
    f = np.stack(planes, -1) * np.float32(0.731) + rng.uniform(-3.0, 3.0, (h, w, c)).astype(np.float32)
    return np.ascontiguousarray(f.astype(np.float32))


def _special(frame, seed):
    """frame with NaN, +-inf, -0 and subnormals in a few pixels and on its border rows and columns."""
    rng = np.random.default_rng(seed)
    f = frame.copy()
    h, w, c = f.shape
    vals = np.array([np.nan, np.inf, -np.inf, -0.0, 1e-41, -3e-39], np.float32)
    m = rng.random((h, w, c)) < 0.004
    f[m] = rng.choice(vals, int(m.sum()))
    f[0, ::7, 0] = -0.0
    f[-1, ::5, -1] = np.float32(2e-40)
    f[h // 2, 1, :] = np.inf
    f[3, -1, 0] = np.nan
    return f


def _bits(t):
    return t.contiguous().view(torch.int32)


def _same(x, y):
    """Equal as int32, except that any NaN equals any NaN (the device makes one canonical NaN, the CPU keeps operands')."""
    if x.shape != y.shape:
        return False
    nx, ny = torch.isnan(x), torch.isnan(y)
    return torch.equal(nx, ny) and torch.equal(_bits(x)[~nx], _bits(y)[~ny])


def _equal(a, b):
    assert len(a) == len(b)
    for fa, fb in zip(a, b):
        assert len(fa) == len(fb)
        for x, y in zip(fa, fb):
            assert (x is None) == (y is None)
            if x is not None:
                assert x.shape == y.shape and torch.equal(_bits(x), _bits(y))


def _pyramid(sd, frames, scales, cs, K, variant=1, bil=False):
    return sd.vl_hog_pyramid(frames, scales, cs, K, variant, multichannel=True, bilinear_orientations=bil, float_frames=True)


def _check_levels(sd, frames, feats, sizes, scales, cs, K, variant, bil, same=None):
    """Every level of feats is vl_hog of resize_f32 of its frame; returns the number of empty levels."""
    levels, where, empty = [], [], 0
    for f, frame in enumerate(frames):
        for s, scale in enumerate(scales):
            lw, lh = sizes[f][s]
            assert (lw, lh) == (math.floor(frame.shape[1] * scale + 0.5), math.floor(frame.shape[0] * scale + 0.5))
            (_, _), (dd, hh, hw) = sd.hog_pyramid_shape(frame.shape[1], frame.shape[0], scale, cs, K, variant)
            if hw == 0:
                assert feats[f][s] is None
                empty += 1
                continue
            levels.append(resize_f32(frame, lw, lh))
            where.append((f, s, (dd, hh, hw)))
    ref = sd.vl_hog(levels, cs, K, variant, bilinear_orientations=bil, channels_last=True)
    for (f, s, shape), r in zip(where, ref):
        assert tuple(feats[f][s].shape) == shape == tuple(r.shape)
        if same is None:
            assert torch.equal(_bits(feats[f][s]), _bits(r)), (f, scales[s])
        else:
            assert same(feats[f][s], r), (f, scales[s])
    return empty


@pytest.mark.parametrize("c", [1, 3, 4, 16])
@pytest.mark.parametrize("bil", [False, True])
@pytest.mark.parametrize("variant", [0, 1])
@pytest.mark.parametrize("cs,K", [(8, 9), (4, 4), (11, 16)])
def test_levels_are_dense_images_of_the_restated_resize(sd, c, bil, variant, cs, K):
    frames = [_frame(97, 131, c, 1), _frame(45, 61, c, 2), _frame(13, 200, c, 3)]
    feats, sizes = _pyramid(sd, frames, SCALES, cs, K, variant, bil)
    assert _check_levels(sd, frames, feats, sizes, SCALES, cs, K, variant, bil) > 0


@pytest.mark.parametrize("c", [1, 3, 4])
@pytest.mark.parametrize("bil", [False, True])
def test_non_finite_and_subnormal_pixels(sd, c, bil):
    frames = [_special(_frame(97, 131, c, 4), 5), _special(_frame(60, 64, c, 6), 7)]
    scales = SCALES + [3.0, 1.0 / 3.0]
    for cs, K, variant in [(8, 9, 1), (4, 4, 0)]:
        feats, sizes = _pyramid(sd, frames, scales, cs, K, variant, bil)
        _check_levels(sd, frames, feats, sizes, scales, cs, K, variant, bil, same=_same)
    # the resized levels carry NaN and inf into the features' input, zero-weight taps included (inf * 0)
    lv = [resize_f32(f, *sizes[i][s]) for i, f in enumerate(frames) for s, sc in enumerate(scales) if sc != 1.0]
    assert any(np.isnan(v).any() for v in lv) and any(np.isinf(v).any() for v in lv)


@pytest.mark.parametrize("c", [1, 3])
def test_integer_frames_give_the_8bit_levels(sd, c):
    u8 = [np.ascontiguousarray(np.stack([synth.smooth_images(1, h, w, seed=s + k, sigma=1.0)[0] for k in range(c)], -1))
          for s, (h, w) in enumerate([(97, 131), (120, 160), (45, 61)])]
    fl = [f.astype(np.float32) for f in u8]
    for cs, K, variant in [(8, 9, 1), (4, 16, 0)]:
        # the level of the frame's size is the frame itself, for any 8-bit values
        _equal(_pyramid(sd, fl, [1.0], cs, K, variant)[0], sd.vl_hog_pyramid(u8, [1.0], cs, K, variant, multichannel=True)[0])
        # at exact 2x upscales both rules are exact on multiples of 16: every value is (9a + 3b + 3c + d) / 16
        q = [f & 0xF0 for f in u8]
        _equal(_pyramid(sd, [f.astype(np.float32) for f in q], [1.0, 2.0], cs, K, variant)[0],
               sd.vl_hog_pyramid(q, [1.0, 2.0], cs, K, variant, multichannel=True)[0])


def _raw(sd, data, frame, image_stride, count, channels, scales, cs, K, variant, bil, dtype=1, ptr=None):
    """sd_hog_pyramid_float through the C ABI -> (rc, output buffer with a canary around every level, [(offset, size)])."""
    from superviseddescent_b200 import _capi
    ctx = sd.default_context()
    ib = _capi.HogImagesC()
    ib.d_data, ib.dtype, ib.channels, ib.count = data.data_ptr() if ptr is None else ptr, dtype, channels, count
    ib.frame = _capi.HogImageC(*frame)
    ib.image_stride = image_stride
    ib.d_frames = None
    w, h = frame[0], frame[1]
    offs, pos = [], 7
    for _ in range(max(count, 0)):
        for s in scales:
            try:
                (_, _), (dd, hh, hw) = sd.hog_pyramid_shape(w, h, s, cs, K, variant)
            except Exception:
                dd = hh = hw = 0
            offs.append((pos, dd * hh * hw))
            pos += dd * hh * hw + 5
    out = torch.full((pos + 7,), CANARY, dtype=torch.float32, device="cuda")
    d_off = torch.tensor([o for o, _ in offs] or [0], dtype=torch.int64, device="cuda")
    sc = (C.c_double * len(scales))(*scales)
    rc = _capi.lib().sd_hog_pyramid_float(ctx.h, C.byref(ib), sc, len(scales), cs, K, variant, int(bil), C.c_void_p(out.data_ptr()),
                                          C.c_void_p(d_off.data_ptr()))
    torch.cuda.synchronize()
    return rc, out, offs


@pytest.mark.parametrize("bil", [False, True])
def test_planar_interleaved_and_strided_views_agree(sd, bil):
    n, h, w, c, cs, K, v = 3, 90, 117, 3, 8, 9, 1
    frames = np.stack([_frame(h, w, c, 20 + i) for i in range(n)])
    want = _pyramid(sd, torch.from_numpy(frames).cuda(), SCALES, cs, K, v, bil)[0]
    # strided: rows wider than the pixels and a fourth channel that is not read, read in place
    wide = torch.zeros((n, h, w + 21, c + 1), dtype=torch.float32)
    wide[:, :, :w, :c] = torch.from_numpy(frames)
    wide[:, :, :, c] = float("nan")
    _equal(_pyramid(sd, wide.cuda()[:, :, :w, :c], SCALES, cs, K, v, bil)[0], want)
    _equal(_pyramid(sd, list(frames), SCALES, cs, K, v, bil)[0], want)
    _equal(_pyramid(sd, frames, SCALES, cs, K, v, bil)[0], want)                      # a host batch
    # planar (C, H, W) per frame through the C ABI: pixel stride 1, channel stride H * W; canaries around every level
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
    assert (out[:7] == CANARY).all() and (out[-7:] == CANARY).all()


def test_frames_are_batch_independent(sd):
    frames = [_frame(97, 131, 3, 30), _frame(120, 160, 3, 31), _frame(45, 61, 3, 32), _frame(13, 200, 3, 33)]
    for bil in (False, True):
        together = _pyramid(sd, frames, SCALES, 8, 9, 1, bil)[0]
        for f, frame in enumerate(frames):
            _equal([together[f]], _pyramid(sd, [frame], SCALES, 8, 9, 1, bil)[0])
        _equal(_pyramid(sd, frames[::-1], SCALES, 8, 9, 1, bil)[0][::-1], together)


def test_batch_over_several_scratch_slices(sd):
    # 640 x 480 x 3 floats at scales 4, 1 and 0.5 are 63.6 MB of levels: each frame fills a 64 MiB slice of its own, so four
    # frames of different sizes take four slices
    frames = [_frame(480 - 8 * i, 640 - 12 * i, 3, 40 + i) for i in range(4)]
    scales = [4.0, 1.0, 0.5]
    ctx = sd.default_context()
    before = ctx.launches()
    together = _pyramid(sd, frames, scales, 8, 9, 1)[0]
    torch.cuda.synchronize()
    launches = ctx.launches() - before
    assert launches >= 2 * 3, launches                          # a resize and a HOG launch per slice
    for f, frame in enumerate(frames):
        _equal([together[f]], _pyramid(sd, [frame], scales, 8, 9, 1)[0])


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_ref
    vl_hog_ref.build()
    if not vl_hog_ref.available():
        pytest.fail("oracle/_ref (the reference's hog.c with channels) is not built: run build()")
    return vl_hog_ref


@pytest.mark.parametrize("bil", [False, True])
def test_levels_within_hog_c_bar_on_restated_levels(sd, ref, bil):
    frame = _frame(120, 160, 3, 50)
    worst = 0.0
    for cs, K, variant in [(8, 9, 1), (4, 4, 0), (11, 16, 1)]:
        feats, sizes = _pyramid(sd, [frame], SCALES, cs, K, variant, bil)
        for s in range(len(SCALES)):
            if feats[0][s] is None:
                continue
            lw, lh = sizes[0][s]
            lvl = resize_f32(frame, lw, lh)
            want = ref.vl_hog(np.ascontiguousarray(lvl.transpose(2, 0, 1)), cs, K, variant, bil)
            e = rel_err(feats[0][s].cpu().numpy(), want)
            worst = max(worst, e)
            assert e <= 1e-4, (cs, K, variant, SCALES[s], e)
    print(f"float pyramid against hog.c: worst rel err {worst:.2e}")


def test_refusals_write_nothing(sd):
    from superviseddescent_b200 import _capi
    h, w = 40, 50
    f32 = torch.from_numpy(_frame(h, w, 3, 60)).cuda()
    u8 = f32.clamp(0, 255).to(torch.uint8)
    hwc = (w, h, 0, 3 * w, 3, 1)
    cases = [dict(data=u8, dtype=0), dict(dtype=7), dict(ptr=f32.data_ptr() + 2), dict(channels=0), dict(channels=17),
             dict(scales=[0.0]), dict(scales=[4.5]), dict(scales=[1.0, float("nan")]), dict(frame=(w, h, 0, -3 * w, 3, 1)),
             dict(frame=(w, h, 0, 3 * w, -3, 1)), dict(frame=(w, h, 0, 3 * w, 3, -1)), dict(frame=(w, h, -1, 3 * w, 3, 1)),
             dict(frame=(0, h, 0, 3 * w, 3, 1)), dict(image_stride=-1, count=2), dict(bil=2)]
    for kw in cases:
        a = dict(data=f32, frame=hwc, image_stride=0, count=1, channels=3, scales=[1.0, 0.5], bil=0, dtype=1, ptr=None)
        a.update(kw)
        rc, out, _ = _raw(sd, a["data"], a["frame"], a["image_stride"], a["count"], a["channels"], a["scales"], 8, 9, 1, a["bil"],
                          a["dtype"], a["ptr"])
        print("refused:", kw, _capi.lib().sd_last_error(sd.default_context().h).decode())
        assert rc == 1, kw
        assert (out == CANARY).all(), kw
    # the 8-bit pyramid keeps refusing float frames, and the float pyramid is reached through float_frames only
    with pytest.raises(sd.SdError):
        sd.vl_hog_pyramid(f32[None], [1.0], 8, 9, 1, multichannel=True)
    with pytest.raises(ValueError):
        sd.vl_hog_pyramid(f32[None], [1.0], 8, 9, 1, float_frames=True)
    with pytest.raises(ValueError):
        sd.vl_hog_pyramid(u8[None], [1.0], 8, 9, 1, multichannel=True, float_frames=True)

"""Dense HOG of whole frames on the device (sd_hog_dense, api.hog_dense) against the reference's own hog.c (oracle/_ref), against
the landmark-patch kernel, and for batch independence, host-frame upload and argument checks."""
import ctypes as C

import numpy as np
import pytest

import synth
from colour_examples import bgr_with_gray
from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _frame(h, w, seed):
    """Smooth structure plus noise plus flat areas: large and small gradients, zero gradients and exact ties."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 127.5 + 90 * np.sin(x / 13.0 + np.cos(y / 17.0)) * np.cos(y / 9.0) + rng.normal(0, 12, (h, w))
    img = np.clip(np.round(img), 0, 255).astype(np.uint8)
    img[h // 3:h // 3 + max(1, h // 8), :] = 77                    # a flat band
    return img


def _ref_hog(oracle, img, cs, K, variant):
    """vl_hog_put_image + vl_hog_extract of the reference (oracle/_ref): features (dd, hogH, hogW)."""
    r = oracle.ref()
    f = np.ascontiguousarray(img, dtype=np.float32)
    h, w = f.shape
    dims = (C.c_int * 3)()
    fp = f.ctypes.data_as(C.POINTER(C.c_float))
    assert r.ref_vl_hog(variant, K, fp, w, h, cs, None, dims) == 0
    out = np.zeros((dims[2], dims[1], dims[0]), dtype=np.float32)
    assert r.ref_vl_hog(variant, K, fp, w, h, cs, out.ctypes.data_as(C.POINTER(C.c_float)), dims) == 0
    return out


@pytest.fixture(scope="module")
def ref(oracle):
    if not oracle.ref_available():
        pytest.fail("oracle/_ref (the reference's hog.c) is not built: run build()")
    return oracle


@pytest.mark.parametrize("h,w", [(4, 4), (7, 5), (29, 37), (480, 640), (720, 1280), (1080, 1920)])
def test_dense_hog_matches_reference_hog(sd, ref, h, w):
    import torch
    img = _frame(h, w, seed=h + w)
    frames = torch.from_numpy(np.stack([img, img[::-1].copy()])).cuda()
    worst = 0.0
    for cs in (4, 6, 8, 11):
        if (w + cs // 2) // cs == 0 or (h + cs // 2) // cs == 0:
            with pytest.raises(sd.SdError):
                sd.hog_dense(frames, cs, 4, 1)
            continue
        for K in (4, 9):
            for variant in (0, 1):
                got = sd.hog_dense(frames, cs, K, variant).cpu().numpy()
                for i in range(2):
                    want = _ref_hog(ref, frames[i].cpu().numpy(), cs, K, variant)
                    assert got[i].shape == want.shape, (h, w, cs, K, variant)
                    e = rel_err(got[i], want)
                    worst = max(worst, e)
                    assert e <= TOL, (h, w, cs, K, variant, e)
    print(f"dense HOG {w} x {h}: worst rel err against hog.c {worst:.2e}")


@pytest.mark.parametrize("cs,K,variant", [(32, 16, 1), (1, 1, 0), (2, 3, 1), (17, 16, 0)])
def test_dense_hog_matches_reference_hog_at_the_ends_of_the_range(sd, ref, cs, K, variant):
    """The extremes of the supported range (cell size 1..32, K 1..16, the generic-K kernel): K = 1 leaves the gx = 0 axis
    unvoted, as hog.c does."""
    import torch
    img = _frame(75, 101, seed=cs * K)
    got = sd.hog_dense(torch.from_numpy(img[None].copy()).cuda(), cs, K, variant).cpu().numpy()[0]
    want = _ref_hog(ref, img, cs, K, variant)
    assert got.shape == want.shape
    e = rel_err(got, want)
    print(f"dense HOG cs {cs} K {K} variant {variant}: rel err against hog.c {e:.2e}")
    assert e <= TOL


@pytest.mark.parametrize("cs", [6, 8, 10])
@pytest.mark.parametrize("K", [4, 9])
@pytest.mark.parametrize("variant", [0, 1])
def test_dense_hog_of_a_window_equals_the_fixed_patch_row(sd, cs, K, variant):
    """A window of fs x fs pixels cut from a frame gives, bit for bit, the features of the fixed-patch HogTransform (sd_hog_batch)
    for a landmark at the window's centre, after undoing the row's per-dimension transpose ([dim][cell col][cell row])."""
    import torch
    nc = 5
    fs, half = nc * cs, nc * (cs // 2)
    img = _frame(160, 200, seed=cs * 100 + K)
    rng = np.random.default_rng(cs + K + variant)
    L = 6
    cx = rng.integers(half, 200 - half + 1, L)
    cy = rng.integers(half, 160 - half + 1, L)
    x = np.concatenate([cx, cy]).astype(np.float32).reshape(1, -1).copy()
    row = sd.FixedHogTransform(img[None], variant, nc, cs, K)(x, 0).cpu().numpy()[0]
    windows = np.stack([img[y - half:y + half, xx - half:xx + half] for xx, y in zip(cx, cy)])
    dense = sd.hog_dense(torch.from_numpy(windows).cuda(), cs, K, variant).cpu().numpy()
    dd = 3 * K + 4 if variant == 1 else 4 * K
    assert dense.shape == (L, dd, nc, nc) and row.size == L * dd * nc * nc
    for l in range(L):
        assert np.array_equal(dense[l].transpose(0, 2, 1).ravel(), row[l * dd * nc * nc:(l + 1) * dd * nc * nc]), l
    assert fs == windows.shape[1]


def _dense_into(sd, ctx, ib, cs, K, variant, out, offsets):
    from superviseddescent_b200 import _capi
    return _capi.lib().sd_hog_dense(ctx.h, C.byref(ib), cs, K, variant, _capi.ptr(out), _capi.ptr(offsets))


@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (4, 4, 0), (11, 9, 1), (3, 7, 0)])
def test_dense_hog_batches_are_frame_independent(sd, cs, K, variant):
    """Mixed sizes (per-frame descriptors, caller offsets with gaps) and one size (a device tensor, NULL offsets): every frame's
    output is bit-identical to the frame computed alone, the floats around and between the blocks are untouched, and two runs are
    bit-identical."""
    import torch
    ctx = sd.default_context()
    sizes = [(97, 131), (64, 48), (130, 203), (33, 40), (97, 131)]
    frames = [_frame(h, w, seed=7 * i) for i, (h, w) in enumerate(sizes)]
    alone = [sd.hog_dense([f], cs, K, variant)[0] for f in frames]
    for a, f in zip(alone, frames):
        assert tuple(a.shape) == sd.hog_dense_shape(f.shape[1], f.shape[0], cs, K, variant)
    buf, ib = sd._upload_host_frames([sd._host_frame(f)[0] for f in frames], ctx)
    assert ib.d_frames
    gap = 5
    starts, pos = [], gap
    for a in alone:
        starts.append(pos)
        pos += a.numel() + gap
    sentinel = -1234.5
    offsets = torch.tensor(starts, dtype=torch.int64, device="cuda")
    runs = []
    for _ in range(2):
        out = torch.full((pos,), sentinel, dtype=torch.float32, device="cuda")
        assert _dense_into(sd, ctx, ib, cs, K, variant, out, offsets) == 0
        runs.append(out.cpu().numpy())
    assert np.array_equal(runs[0], runs[1])
    got = runs[0]
    mask = np.ones(pos, dtype=bool)
    for s, a in zip(starts, alone):
        assert np.array_equal(got[s:s + a.numel()], a.cpu().numpy().ravel())
        mask[s:s + a.numel()] = False
    assert np.all(got[mask] == sentinel)
    # frames of different sizes without offsets are refused
    assert _dense_into(sd, ctx, ib, cs, K, variant, torch.empty(pos, device="cuda"), None) == 1
    # one size: a strided device batch with NULL offsets (frame i at i * dd * hogH * hogW), and 16-byte aligned rows (the TMA path)
    for w in (131, 144):
        eq = torch.from_numpy(np.stack([_frame(97, w, seed=50 + i) for i in range(6)])).cuda()
        single = [sd.hog_dense(eq[i:i + 1], cs, K, variant)[0] for i in range(6)]
        from superviseddescent_b200._capi import ImageBatchC
        ib1 = ImageBatchC(C.c_void_p(eq.data_ptr()), w, 97, eq.stride(1), eq.stride(0), 6)
        per = single[0].numel()
        out = torch.full((6 * per + gap,), sentinel, dtype=torch.float32, device="cuda")
        assert _dense_into(sd, ctx, ib1, cs, K, variant, out, None) == 0
        got = out.cpu().numpy()
        for i in range(6):
            assert np.array_equal(got[i * per:(i + 1) * per], single[i].cpu().numpy().ravel()), (w, i)
        assert np.all(got[6 * per:] == sentinel)
        # the same frames uploaded from the host (rows at a 16-byte pitch: the TMA route) give what the device batch gives
        host = sd.hog_dense([eq[i].cpu().numpy() for i in range(6)], cs, K, variant)
        assert np.array_equal(host.cpu().numpy().ravel(), got[:6 * per]), w


def test_dense_hog_of_host_frames(sd):
    """Grey and B,G,R numpy frames of different sizes (one of them with a padded row step) equal the device call on the grey frames
    that bgr2gray gives."""
    import torch
    rng = np.random.default_rng(3)
    sizes = [(120, 160), (97, 131), (200, 150), (64, 64)]
    grey = [synth.smooth_images(1, h, w, seed=70 + i)[0] for i, (h, w) in enumerate(sizes)]
    colour = [bgr_with_gray(g, rng.integers(-40, 41, g.shape), rng.integers(-40, 41, g.shape)) for g in grey]
    padded = np.zeros((97, 136, 3), dtype=np.uint8)
    padded[:, :131] = colour[1]
    colour[1] = padded[:, :131]
    mixed = [colour[0], grey[1], colour[2], grey[3]]
    for cs, K, variant in ((8, 9, 1), (6, 4, 0)):
        for frames in (grey, colour, mixed):
            got = sd.hog_dense(frames, cs, K, variant)
            assert isinstance(got, list) and len(got) == 4
            for i, f in enumerate(frames):
                g = sd.bgr2gray(f[None]) if f.ndim == 3 else torch.from_numpy(f[None].copy()).cuda()
                want = sd.hog_dense(g, cs, K, variant)[0]
                assert np.array_equal(got[i].cpu().numpy(), want.cpu().numpy()), (cs, K, i)
        same = sd.hog_dense(np.stack([colour[0], colour[0]]), cs, K, variant)
        assert tuple(same.shape[:1]) == (2,) and np.array_equal(same[1].cpu().numpy(), sd.hog_dense([grey[0]], cs, K, variant)[0].cpu().numpy())


def test_dense_hog_invalid_arguments(sd):
    """Every invalid case is SD_ERR_INVALID and queues no kernel."""
    import torch
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import FrameC, ImageBatchC
    ctx = sd.default_context()
    lib = _capi.lib()
    img = torch.zeros((2, 40, 48), dtype=torch.uint8, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")

    def batch(w=48, h=40, **kw):
        return ImageBatchC(C.c_void_p(img.data_ptr()), w, h, 48, 40 * 48, 2, **kw)

    roi = torch.zeros(64, dtype=torch.uint8, device="cuda")
    cases = [(batch(w=3), 4, 4, 1), (batch(h=3), 4, 4, 1), (batch(w=4), 11, 4, 1), (batch(h=4), 11, 4, 0),
             (batch(), 4, 0, 1), (batch(), 4, 17, 1), (batch(), 0, 4, 1), (batch(), 33, 4, 1), (batch(), 4, 4, 2),
             (batch(), 4, 4, -1), (batch(d_roi=C.c_void_p(roi.data_ptr())), 4, 4, 1)]
    # a descriptor table with one frame that is too small
    table = (FrameC * 2)(FrameC(48, 40, 48, 0, 0), FrameC(3, 40, 48, 0, 1920))
    d_table = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    cases.append((batch(d_frames=C.c_void_p(d_table.data_ptr())), 4, 4, 1))
    torch.cuda.synchronize()
    before = ctx.launches()
    for ib, cs, K, variant in cases:
        assert lib.sd_hog_dense(ctx.h, C.byref(ib), cs, K, variant, _capi.ptr(out), None) == 1, (ib.width, ib.height, cs, K, variant)
    assert ctx.launches() == before
    assert not torch.any(out != 0)
    w, h, d = C.c_int(), C.c_int(), C.c_int()
    for args in ((3, 40, 4, 4, 1), (40, 3, 4, 4, 1), (4, 40, 11, 4, 1), (40, 40, 4, 0, 1), (40, 40, 4, 17, 1), (40, 40, 0, 4, 1),
                 (40, 40, 33, 4, 1), (40, 40, 4, 4, 2)):
        assert lib.sd_hog_dense_shape(*args, C.byref(w), C.byref(h), C.byref(d)) == 1, args
    assert lib.sd_hog_dense_shape(4, 4, 1, 16, 0, C.byref(w), C.byref(h), C.byref(d)) == 0 and (w.value, h.value, d.value) == (4, 4, 64)
    assert lib.sd_hog_dense_shape(40, 40, 32, 1, 1, C.byref(w), C.byref(h), C.byref(d)) == 0 and (w.value, h.value, d.value) == (1, 1, 7)

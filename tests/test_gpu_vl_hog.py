"""Dense HOG of 8-bit and float frames of one or more channels, nearest-bin and bilinear orientations (sd_hog_dense_images,
api.vl_hog), against the reference's own hog.c (oracle/_ref), against the 8-bit grey path (sd_hog_dense), and for layouts, batch
independence, host input and argument checks."""
import ctypes as C

import numpy as np
import pytest

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _texture(h, w, seed):
    """Smooth structure plus noise plus a flat band: large and small gradients, zero gradients and exact ties (values 0..255)."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = 127.5 + 90 * np.sin(x / (9.0 + seed % 7) + np.cos(y / 17.0)) * np.cos(y / (5.0 + seed % 5)) + rng.normal(0, 12, (h, w))
    img = np.clip(np.round(img), 0, 255)
    img[h // 3:h // 3 + max(1, h // 8), :] = 77
    return img


def _frames(kind, c, h, w, seed):
    """(c, h, w) planar frame: 'u8', 'f255' (floats in [0, 255], not integers) or 'f1' (floats in [0, 1])."""
    planes = np.stack([_texture(h, w, seed + 13 * k) for k in range(c)])
    if kind == "u8":
        return planes.astype(np.uint8)
    rng = np.random.default_rng(seed)
    f = np.clip(planes + rng.uniform(-0.5, 0.5, planes.shape), 0, 255).astype(np.float32)
    return f if kind == "f255" else (f / np.float32(255)).astype(np.float32)


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_ref
    vl_hog_ref.build()
    if not vl_hog_ref.available():
        pytest.fail("oracle/_ref (the reference's hog.c with channels) is not built: run build()")
    return vl_hog_ref


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("h,w", [(4, 4), (7, 5), (29, 37), (480, 640), (1080, 1920)])
@pytest.mark.parametrize("kind", ["u8", "f255", "f1"])
def test_vl_hog_matches_reference_hog(sd, ref, h, w, kind):
    worst = 0.0
    for c in (1, 3):
        frame = _frames(kind, c, h, w, seed=h + w + c)
        batch = _dev(frame[None])
        for cs in (4, 8, 11):
            if (w + cs // 2) // cs == 0 or (h + cs // 2) // cs == 0:
                with pytest.raises(sd.SdError):
                    sd.vl_hog(batch, cs, 4, 1)
                continue
            for K in (4, 9):
                for variant in (0, 1):
                    for bil in (False, True):
                        got = sd.vl_hog(batch, cs, K, variant, bilinear_orientations=bil).cpu().numpy()[0]
                        want = ref.vl_hog(frame.astype(np.float32), cs, K, variant, bil)
                        assert got.shape == want.shape
                        e = rel_err(got, want)
                        worst = max(worst, e)
                        assert e <= TOL, (kind, c, h, w, cs, K, variant, bil, e)
    print(f"vl_hog {kind} {w} x {h}: worst rel err against hog.c {worst:.2e}")


@pytest.mark.parametrize("cs,K,variant,c", [(32, 16, 1, 3), (1, 1, 0, 3), (2, 3, 1, 16), (17, 16, 0, 16), (32, 1, 1, 1), (1, 16, 0, 1)])
@pytest.mark.parametrize("kind", ["u8", "f1"])
@pytest.mark.parametrize("bil", [False, True])
def test_vl_hog_matches_reference_hog_at_the_ends_of_the_range(sd, ref, cs, K, variant, c, kind, bil):
    frame = _frames(kind, c, 75, 101, seed=cs * K + c)
    got = sd.vl_hog(_dev(frame[None]), cs, K, variant, bilinear_orientations=bil).cpu().numpy()[0]
    want = ref.vl_hog(frame.astype(np.float32), cs, K, variant, bil)
    e = rel_err(got, want)
    print(f"vl_hog cs {cs} K {K} variant {variant} channels {c} {kind} bilinear {bil}: rel err against hog.c {e:.2e}")
    assert got.shape == want.shape and e <= TOL


@pytest.mark.parametrize("scale", [1e-12, 1e-21])
@pytest.mark.parametrize("bil", [False, True])
def test_vl_hog_of_moduli_below_the_floor(sd, ref, scale, bil):
    """Gradient moduli below 1e-10 (the unit vector divides by the 1e-10 floor), and at 1e-21 squares that are subnormal."""
    frame = (_frames("f1", 3, 61, 83, seed=5) * np.float32(scale)).astype(np.float32)
    for cs, K, variant in ((4, 9, 1), (8, 4, 0)):
        got = sd.vl_hog(_dev(frame[None]), cs, K, variant, bilinear_orientations=bil).cpu().numpy()[0]
        want = ref.vl_hog(frame, cs, K, variant, bil)
        e = rel_err(got, want)
        print(f"vl_hog moduli x {scale:g} cs {cs} K {K} bilinear {bil}: max |f| {np.abs(want).max():.2e}, rel err {e:.2e}")
        assert np.abs(want).max() > 0 and e <= TOL


@pytest.mark.parametrize("cs,K,variant", [(8, 9, 1), (4, 4, 0), (11, 9, 1), (3, 7, 0)])
def test_vl_hog_bit_identities(sd, cs, K, variant):
    """u8 grey nearest-bin equals sd_hog_dense on its TMA route (rows a multiple of 16 bytes) and its load-loop route, whether
    the new entry hands the frames to that kernel or computes them itself (a column-major view); a float frame holding a u8 frame's
    values equals the u8 result, nearest-bin and bilinear; identical channels (copies, or a zero channel stride) equal one
    channel; planar, interleaved and a strided view read in place agree."""
    import torch
    for w in (144, 131):
        grey = np.stack([_texture(97, w, seed=i + w).astype(np.uint8) for i in range(3)])
        g = _dev(grey)
        want = sd.hog_dense(g, cs, K, variant)
        assert torch.equal(sd.vl_hog(g, cs, K, variant), want)
        colmajor = g.transpose(1, 2).contiguous().transpose(1, 2)
        assert colmajor.stride(2) != 1
        assert torch.equal(sd.vl_hog(colmajor, cs, K, variant), want)
        for bil in (False, True):
            u8 = sd.vl_hog(colmajor, cs, K, variant, bilinear_orientations=bil)
            assert torch.equal(sd.vl_hog(g.float(), cs, K, variant, bilinear_orientations=bil), u8), (w, bil)
            for c in (3, 16):
                assert torch.equal(sd.vl_hog(g[:, None].expand(3, c, 97, w), cs, K, variant, bilinear_orientations=bil), u8), (w, c)
            assert torch.equal(sd.vl_hog(g[:, None].repeat(1, 3, 1, 1).float(), cs, K, variant, bilinear_orientations=bil), u8)
    for kind in ("u8", "f1"):
        planar = np.stack([_frames(kind, 3, 70, 90, seed=20 + i) for i in range(2)])
        for bil in (False, True):
            p = sd.vl_hog(_dev(planar), cs, K, variant, bilinear_orientations=bil)
            inter = sd.vl_hog(_dev(planar.transpose(0, 2, 3, 1)), cs, K, variant, bilinear_orientations=bil, channels_last=True)
            assert torch.equal(p, inter), (kind, bil)
            # a strided view: every other row and column of a larger planar buffer, channels in reverse order
            big = np.zeros((2, 3, 140, 180), dtype=planar.dtype)
            big[:, ::-1, ::2, ::2] = planar
            view = _dev(big).flip(1)[:, :, ::2, ::2]
            assert view.stride(2) == 360 and view.stride(3) == 2
            assert torch.equal(sd.vl_hog(view, cs, K, variant, bilinear_orientations=bil), p), (kind, bil)


@pytest.mark.parametrize("bil", [False, True])
def test_vl_hog_channel_ties(sd, bil):
    """Channels (I, 255 - I) give hog(I) and (255 - I, I) give hog(255 - I) bit for bit (the first channel keeps a tie); under
    UoCTTI the directed halves of the two are swapped and the rest equal, under Dalal-Triggs every dimension is equal."""
    import torch
    for dtype in (np.uint8, np.float32):                           # integer values: 255 - I is exact in float
        img = _frames("u8", 1, 83, 101, seed=9)[0].astype(dtype)
        inv = (dtype(255) - img).astype(dtype)
        for cs, K in ((8, 9), (4, 4)):
            hi = {v: sd.vl_hog(_dev(img[None]), cs, K, v, bilinear_orientations=bil)[0] for v in (0, 1)}
            hn = {v: sd.vl_hog(_dev(inv[None]), cs, K, v, bilinear_orientations=bil)[0] for v in (0, 1)}
            for v in (0, 1):
                assert torch.equal(sd.vl_hog(_dev(np.stack([img, inv])[None]), cs, K, v, bilinear_orientations=bil)[0], hi[v])
                assert torch.equal(sd.vl_hog(_dev(np.stack([inv, img])[None]), cs, K, v, bilinear_orientations=bil)[0], hn[v])
            a, b = hi[1], hn[1]
            assert torch.equal(a[:K], b[K:2 * K]) and torch.equal(a[K:2 * K], b[:K]) and torch.equal(a[2 * K:], b[2 * K:])
            assert torch.equal(hi[0], hn[0])


def _images_into(sd, ctx, ib, cs, K, variant, bil, out, offsets):
    from superviseddescent_b200 import _capi
    return _capi.lib().sd_hog_dense_images(ctx.h, C.byref(ib), cs, K, variant, bil, _capi.ptr(out), _capi.ptr(offsets))


@pytest.mark.parametrize("cs,K,variant,bil", [(8, 9, 1, 0), (4, 4, 0, 1), (11, 9, 1, 1), (3, 7, 0, 0)])
@pytest.mark.parametrize("kind", ["u8", "f1"])
def test_vl_hog_batches_are_frame_independent(sd, cs, K, variant, bil, kind):
    """Mixed sizes and layouts through a descriptor table with caller offsets that leave gaps, and one size with NULL offsets:
    every frame equals the frame computed alone, the floats around the blocks are untouched, and two runs are bit-identical."""
    import torch
    from superviseddescent_b200._capi import HogImageC, HogImagesC
    ctx = sd.default_context()
    sizes = [(97, 131), (64, 48), (130, 203), (33, 40), (97, 131)]
    frames = [_frames(kind, 3, h, w, seed=7 * i) for i, (h, w) in enumerate(sizes)]
    alone = [sd.vl_hog(_dev(f[None]), cs, K, variant, bilinear_orientations=bool(bil))[0] for f in frames]
    # frames 1 and 3 interleaved, the others planar, packed with gaps
    parts, descs, pos = [], [], 3
    for i, f in enumerate(frames):
        c, h, w = f.shape
        inter = i % 2 == 1
        data = f.transpose(1, 2, 0).ravel() if inter else f.ravel()
        descs.append(HogImageC(w, h, pos, w * c if inter else w, c if inter else 1, 1 if inter else h * w))
        parts += [np.zeros(3, f.dtype) if i == 0 else np.zeros(5, f.dtype), data]
        pos += data.size + 5
    buf = _dev(np.concatenate([np.zeros(0, frames[0].dtype)] + parts))
    table = (HogImageC * len(descs))(*descs)
    d_table = _dev(np.frombuffer(bytes(table), dtype=np.uint8).copy())
    ib = HogImagesC(C.c_void_p(buf.data_ptr()), 0 if kind == "u8" else 1, 3, len(frames), HogImageC(), 0, C.c_void_p(d_table.data_ptr()))
    gap, sentinel = 5, -1234.5
    starts, p = [], gap
    for a in alone:
        starts.append(p)
        p += a.numel() + gap
    offsets = torch.tensor(starts, dtype=torch.int64, device="cuda")
    runs = []
    for _ in range(2):
        out = torch.full((p,), sentinel, dtype=torch.float32, device="cuda")
        assert _images_into(sd, ctx, ib, cs, K, variant, bil, out, offsets) == 0
        runs.append(out.cpu().numpy())
    assert np.array_equal(runs[0], runs[1])
    mask = np.ones(p, dtype=bool)
    for s, a in zip(starts, alone):
        assert np.array_equal(runs[0][s:s + a.numel()], a.cpu().numpy().ravel())
        mask[s:s + a.numel()] = False
    assert np.all(runs[0][mask] == sentinel)
    assert _images_into(sd, ctx, ib, cs, K, variant, bil, torch.empty(p, device="cuda"), None) == 1
    # one size, NULL offsets: frame i at i * dd * hogH * hogW
    eq = np.stack([_frames(kind, 3, 97, 131, seed=50 + i) for i in range(6)])
    single = [sd.vl_hog(_dev(eq[i:i + 1]), cs, K, variant, bilinear_orientations=bool(bil))[0] for i in range(6)]
    d = _dev(eq)
    ib1 = HogImagesC(C.c_void_p(d.data_ptr()), 0 if kind == "u8" else 1, 3, 6, HogImageC(131, 97, 0, 131, 1, 97 * 131), 3 * 97 * 131, None)
    per = single[0].numel()
    out = torch.full((6 * per + gap,), sentinel, dtype=torch.float32, device="cuda")
    assert _images_into(sd, ctx, ib1, cs, K, variant, bil, out, None) == 0
    got = out.cpu().numpy()
    for i in range(6):
        assert np.array_equal(got[i * per:(i + 1) * per], single[i].cpu().numpy().ravel()), i
    assert np.all(got[6 * per:] == sentinel)


@pytest.mark.parametrize("kind", ["u8", "f1"])
def test_vl_hog_of_host_frames(sd, kind):
    """numpy lists of mixed sizes, planar and interleaved, and host batches, equal the device call frame by frame."""
    import torch
    sizes = [(120, 160), (97, 131), (200, 150), (64, 64)]
    planar = [_frames(kind, 3, h, w, seed=70 + i) for i, (h, w) in enumerate(sizes)]
    for cs, K, variant, bil in ((8, 9, 1, False), (6, 4, 0, True)):
        want = [sd.vl_hog(_dev(f[None]), cs, K, variant, bilinear_orientations=bil)[0] for f in planar]
        got_p = sd.vl_hog(planar, cs, K, variant, bilinear_orientations=bil)
        got_i = sd.vl_hog([f.transpose(1, 2, 0) for f in planar], cs, K, variant, bilinear_orientations=bil, channels_last=True)
        assert isinstance(got_p, list) and len(got_p) == 4 and len(got_i) == 4
        for i in range(4):
            assert torch.equal(got_p[i], want[i]) and torch.equal(got_i[i], want[i]), (cs, K, i)
        grey = [f[0] for f in planar]
        got_g = sd.vl_hog(grey, cs, K, variant, bilinear_orientations=bil)
        for i in range(4):
            assert torch.equal(got_g[i], sd.vl_hog(_dev(grey[i][None]), cs, K, variant, bilinear_orientations=bil)[0])
        same = sd.vl_hog(np.stack([planar[0], planar[0]]), cs, K, variant, bilinear_orientations=bil)
        assert tuple(same.shape[:1]) == (2,) and torch.equal(same[1], want[0])
        same_list = sd.vl_hog([planar[0].transpose(1, 2, 0)] * 2, cs, K, variant, bilinear_orientations=bil, channels_last=True)
        assert torch.equal(same_list[1], want[0])


def test_vl_hog_invalid_arguments(sd):
    """Every invalid case is SD_ERR_INVALID, queues no kernel and leaves out untouched."""
    import torch
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogImageC, HogImagesC
    ctx = sd.default_context()
    lib = _capi.lib()
    img = torch.zeros(3 * 2 * 40 * 48 + 4, dtype=torch.float32, device="cuda")
    out = torch.zeros(1 << 16, dtype=torch.float32, device="cuda")

    def batch(w=48, h=40, off=0, rs=48, ps=1, cst=1920, dtype=1, channels=3, count=2, stride=5760, data=None, frames=None):
        return HogImagesC(C.c_void_p(data if data is not None else img.data_ptr()), dtype, channels, count,
                          HogImageC(w, h, off, rs, ps, cst), stride, C.c_void_p(frames) if frames else None)

    good = HogImageC(48, 40, 0, 48, 1, 1920)
    table = (HogImageC * 2)(good, HogImageC(48, 40, 5760, -48, 1, 1920))
    d_bad_stride = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    table = (HogImageC * 2)(good, HogImageC(3, 40, 5760, 48, 1, 1920))
    d_small = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    table = (HogImageC * 2)(good, HogImageC(48, 40, -1, 48, 1, 1920))
    d_bad_off = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    cases = [(batch(dtype=2), 4, 4, 1, 0), (batch(dtype=-1), 4, 4, 1, 0), (batch(channels=0), 4, 4, 1, 0),
             (batch(channels=17), 4, 4, 1, 0), (batch(data=img.data_ptr() + 2), 4, 4, 1, 0), (batch(rs=-48), 4, 4, 1, 0),
             (batch(ps=-1), 4, 4, 1, 0), (batch(cst=-1920), 4, 4, 1, 0), (batch(off=-1), 4, 4, 1, 0), (batch(stride=-5760), 4, 4, 1, 0),
             (batch(w=3), 4, 4, 1, 0), (batch(h=3), 4, 4, 1, 1), (batch(w=4), 11, 4, 1, 0), (batch(), 4, 0, 1, 0),
             (batch(), 4, 17, 1, 1), (batch(), 0, 4, 1, 0), (batch(), 33, 4, 1, 1), (batch(), 4, 4, 2, 0), (batch(), 4, 4, 1, 2),
             (batch(), 4, 4, 1, -1), (batch(count=-1), 4, 4, 1, 0),
             (batch(frames=d_bad_stride.data_ptr()), 4, 4, 1, 0), (batch(frames=d_small.data_ptr()), 4, 4, 1, 1),
             (batch(frames=d_bad_off.data_ptr()), 4, 4, 1, 0)]
    torch.cuda.synchronize()
    before = ctx.launches()
    for ib, cs, K, variant, bil in cases:
        assert lib.sd_hog_dense_images(ctx.h, C.byref(ib), cs, K, variant, bil, _capi.ptr(out), None) == 1, \
            (ib.dtype, ib.channels, ib.frame.width, ib.frame.height, cs, K, variant, bil)
    assert lib.sd_hog_dense_images(ctx.h, None, 4, 4, 1, 0, _capi.ptr(out), None) == 1
    assert lib.sd_hog_dense_images(ctx.h, C.byref(batch()), 4, 4, 1, 0, None, None) == 1
    # a valid descriptor table of two sizes without offsets
    table = (HogImageC * 2)(good, HogImageC(40, 40, 5760, 40, 1, 1600))
    d_two = torch.from_numpy(np.frombuffer(bytes(table), dtype=np.uint8).copy()).cuda()
    assert lib.sd_hog_dense_images(ctx.h, C.byref(batch(frames=d_two.data_ptr())), 4, 4, 1, 0, _capi.ptr(out), None) == 1
    assert ctx.launches() == before
    assert not torch.any(out != 0)
    with pytest.raises(ValueError):
        sd.vl_hog(np.zeros((2, 40, 48), np.float64), 4, 4)
    with pytest.raises(ValueError):
        sd.vl_hog([np.zeros((40, 48), np.uint8), np.zeros((40, 48), np.float32)], 4, 4)
    with pytest.raises(ValueError):
        sd.vl_hog([np.zeros((3, 40, 48), np.uint8), np.zeros((2, 40, 48), np.uint8)], 4, 4)
    with pytest.raises(sd.SdError):
        sd.vl_hog(np.zeros((1, 17, 40, 48), np.uint8), 4, 4)

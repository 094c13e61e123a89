"""Dense HOG of caller-supplied polar gradient fields (sd_hog_dense_polar, api.vl_hog_polar) against the reference's own
vl_hog_put_polar_field (oracle/_ref), and for the defined cases, layouts, batch independence, host input and argument checks."""
import ctypes as C

import numpy as np
import pytest

from conftest import rel_err
from polar_fields import angle_sweep, one_vote_per_cell, polar_bins, polar_ho, smooth_field

pytestmark = pytest.mark.gpu
TOL = 1e-4
FLAGS = [(v, d, b) for v in (0, 1) for d in (False, True) for b in (False, True)]   # (variant, directed, bilinear)


@pytest.fixture(scope="module")
def ref(oracle):
    from oracle import vl_hog_polar_ref
    vl_hog_polar_ref.build()
    if not vl_hog_polar_ref.available():
        pytest.fail("oracle/_ref (the reference's hog.c) is not built: run build()")
    return vl_hog_polar_ref


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _polar(sd, m, a, cs, K, variant=1, directed=True, bil=False):
    """Features of one (h, w) field on the device, as numpy."""
    return sd.vl_hog_polar(_dev(m[None]), _dev(a[None]), cs, K, variant, directed=directed,
                           bilinear_orientations=bil).cpu().numpy()[0]


@pytest.mark.parametrize("h,w", [(4, 4), (7, 5), (29, 37), (480, 640), (1080, 1920)])
def test_vl_hog_polar_matches_reference_hog(sd, ref, h, w):
    """Every cs in {1, 4, 8, 11, 32} and K in {1, 4, 9, 16}; all eight (variant, directed, bilinear) combinations on the small
    fields, two per (cs, K) on the large ones, so that every combination meets every size."""
    m, a = smooth_field(h, w, seed=h + w)
    md, ad = _dev(m[None]), _dev(a[None])
    worst, i = 0.0, 0
    for cs in (1, 4, 8, 11, 32):
        if (w + cs // 2) // cs == 0 or (h + cs // 2) // cs == 0:
            with pytest.raises(sd.SdError):
                sd.vl_hog_polar(md, ad, cs, 4)
            continue
        for K in (1, 4, 9, 16):
            flags = FLAGS if h * w < 10000 else [FLAGS[i % 8], FLAGS[(i + 3) % 8]]
            i += 1
            for variant, directed, bil in flags:
                got = sd.vl_hog_polar(md, ad, cs, K, variant, directed=directed, bilinear_orientations=bil).cpu().numpy()[0]
                want = ref.vl_hog_polar(m, a, cs, K, variant, directed, bil)
                assert got.shape == want.shape
                e = rel_err(got, want)
                worst = max(worst, e)
                assert e <= TOL, (h, w, cs, K, variant, directed, bil, e)
    print(f"vl_hog_polar {w} x {h}: worst rel err against hog.c {worst:.2e}")


@pytest.mark.parametrize("K", [1, 4, 9, 16])
def test_one_vote_per_cell(sd, ref, K):
    """One pixel per cell votes, at angles on exact half steps (ties), exact multiples of the step, magnitudes up to 1e7 and
    negative angles: a wrong bin cannot hide in a sum."""
    angles = angle_sweep(K)
    worst = 0.0
    for cs in (4, 8):
        for seed, (h, w) in enumerate([(64, 72), (37, 53)]):
            perm = np.random.default_rng(seed + cs).permutation(len(angles))
            m, a = one_vote_per_cell(h, w, cs, angles[perm], seed)
            for variant, directed, bil in FLAGS:
                got = _polar(sd, m, a, cs, K, variant, directed, bil)
                want = ref.vl_hog_polar(m, a, cs, K, variant, directed, bil)
                e = rel_err(got, want)
                worst = max(worst, e)
                assert e <= TOL, (K, cs, h, w, variant, directed, bil, e)
    print(f"vl_hog_polar one vote per cell, K {K}: worst rel err against hog.c {worst:.2e}")


@pytest.mark.parametrize("h,w", [(29, 37), (64, 48)])
def test_border_pixels_vote(sd, ref, h, w):
    m, a = smooth_field(h, w, seed=3)
    keep = np.zeros((h, w), bool)
    keep[0, :] = keep[-1, :] = keep[:, 0] = keep[:, -1] = True
    m = np.where(keep, np.abs(m) + np.float32(0.5), np.float32(0)).astype(np.float32)
    for cs, K in ((4, 9), (8, 4), (11, 16)):
        for variant, directed, bil in FLAGS:
            got = _polar(sd, m, a, cs, K, variant, directed, bil)
            want = ref.vl_hog_polar(m, a, cs, K, variant, directed, bil)
            assert np.any(want != 0) and np.any(got != 0)
            assert rel_err(got, want) <= TOL, (cs, K, variant, directed, bil)


@pytest.mark.parametrize("cs,K", [(8, 9), (4, 4), (11, 16), (3, 1)])
def test_vl_hog_polar_defined_cases(sd, cs, K):
    """Moduli <= 0 (negative, -0, -inf) give the features of a modulus of 0; non-finite angles (NaN, +-inf) and angles whose
    quotient overflows float give the features of a modulus of 0 there, all finite; |ho| >= 2^63 votes into the exact
    residue, the bin of an angle inside it."""
    h, w = 53, 67
    m, a = smooth_field(h, w, seed=cs + K)
    rng = np.random.default_rng(K)
    m = np.where(m > 0, m, np.float32(0)).astype(np.float32)
    for variant, directed, bil in FLAGS:
        base = _polar(sd, m, a, cs, K, variant, directed, bil)
        neg = m.copy()
        pick = rng.random((h, w)) < 0.2
        neg[pick] = rng.choice(np.array([-1.0, -0.0, -np.inf, -1e-30], np.float32), pick.sum())
        m0 = np.where(pick, np.float32(0), m).astype(np.float32)
        assert np.array_equal(_polar(sd, neg, a, cs, K, variant, directed, bil), _polar(sd, m0, a, cs, K, variant, directed, bil))
        bad = a.copy()
        pick = rng.random((h, w)) < 0.1
        overflow = [3.4e38, -3.4e38] if K >= 4 else []            # 3.4e38 / (pi / K) overflows float from K = 4 on
        bad[pick] = rng.choice(np.array([np.nan, np.inf, -np.inf] + overflow, np.float32), pick.sum())
        got = _polar(sd, m, bad, cs, K, variant, directed, bil)
        assert np.all(np.isfinite(got))
        assert np.array_equal(got, _polar(sd, np.where(pick, np.float32(0), m).astype(np.float32), a, cs, K, variant, directed, bil))
        assert not np.array_equal(got, base)
    # |ho| >= 2^63: the device's bin is the exact residue (hog.c's long conversion overflows there)
    huge = np.array([1e20, -1e20, 3e25, -7.5e30, 2.0 ** 70, 1e36], np.float32)
    assert np.all(np.abs(polar_ho(huge, K).astype(np.float64)) >= 2.0 ** 63)
    for directed in (False, True):
        near = polar_bins(huge, K, directed)[0]
        centre = np.array([(b + 0.25) * np.pi / K for b in near], np.float32)
        assert np.array_equal(polar_bins(centre, K, directed)[0], near)
        mh = np.zeros((h, w), np.float32)
        ah, ac = np.zeros_like(mh), np.zeros_like(mh)
        for j in range(len(huge)):
            mh[5 + 7 * j, 3 + 9 * j] = 1.0 + j
            ah[5 + 7 * j, 3 + 9 * j] = huge[j]
            ac[5 + 7 * j, 3 + 9 * j] = centre[j]
        want = _polar(sd, mh, ac, cs, K, 1, directed, False)
        assert np.any(want != 0)
        # such an ho is an integer: bilinear gives the residue bin weight 1 and the next bin weight 0, the nearest-bin votes
        for bil in (False, True):
            assert np.array_equal(_polar(sd, mh, ah, cs, K, 1, directed, bil), want), (directed, bil)


@pytest.mark.parametrize("K", [1, 4, 9, 16])
def test_undirected_equals_directed_below_pi(sd, K):
    """Angles in [0, pi - pi / 2K) minus a margin keep ho below K - 0.5: nearest bins are < K either way."""
    h, w = 61, 47
    rng = np.random.default_rng(K)
    m, _ = smooth_field(h, w, seed=K)
    a = rng.uniform(0, np.pi - np.pi / (2 * K) - 1e-3, (h, w)).astype(np.float32)
    assert np.all(polar_ho(a, K) < np.float32(K - 0.5))
    for cs in (4, 8):
        for variant in (0, 1):
            assert np.array_equal(_polar(sd, m, a, cs, K, variant, False), _polar(sd, m, a, cs, K, variant, True))


@pytest.mark.parametrize("cs,K,variant,bil", [(8, 9, 1, False), (4, 4, 0, True), (11, 16, 1, True), (3, 7, 0, False)])
def test_vl_hog_polar_layouts(sd, cs, K, variant, bil):
    """Separate planes, one interleaved (count, H, W, 2) buffer and strided views of a larger buffer, all read in place."""
    import torch
    fields = [smooth_field(70, 90, seed=20 + i) for i in range(3)]
    m = np.stack([f[0] for f in fields])
    a = np.stack([f[1] for f in fields])
    for directed in (False, True):
        want = sd.vl_hog_polar(_dev(m), _dev(a), cs, K, variant, directed=directed, bilinear_orientations=bil)
        inter = _dev(np.stack([m, a], axis=-1))
        assert inter[..., 1].data_ptr() == inter[..., 0].data_ptr() + 4
        got = sd.vl_hog_polar(inter[..., 0], inter[..., 1], cs, K, variant, directed=directed, bilinear_orientations=bil)
        assert torch.equal(got, want), directed
        big = np.zeros((2, 3, 140, 180), np.float32)
        big[0, :, ::2, ::2] = m
        big[1, :, ::2, ::2] = a
        bd = _dev(big)
        view_m, view_a = bd[0, :, ::2, ::2], bd[1, :, ::2, ::2]
        assert view_m.stride() == (25200, 360, 2)
        got = sd.vl_hog_polar(view_m, view_a, cs, K, variant, directed=directed, bilinear_orientations=bil)
        assert torch.equal(got, want), directed


def _polar_into(ctx, fb, cs, K, variant, directed, bil, out, offsets):
    from superviseddescent_b200 import _capi
    return _capi.lib().sd_hog_dense_polar(ctx.h, C.byref(fb), cs, K, variant, directed, bil, _capi.ptr(out), _capi.ptr(offsets))


@pytest.mark.parametrize("cs,K,variant,directed,bil", [(8, 9, 1, 1, 0), (4, 4, 0, 0, 1), (11, 9, 1, 0, 1), (3, 7, 0, 1, 0)])
def test_vl_hog_polar_batches_are_field_independent(sd, cs, K, variant, directed, bil):
    """Mixed sizes through a descriptor table with caller offsets that leave gaps, and one size with NULL offsets: every field
    equals the field computed alone, the floats around the blocks are untouched, and two runs are bit-identical."""
    import torch
    from superviseddescent_b200._capi import HogImageC, HogPolarFieldsC
    ctx = sd.default_context()
    sizes = [(97, 131), (64, 48), (130, 203), (33, 40), (97, 131)]
    fields = [smooth_field(h, w, seed=7 * i) for i, (h, w) in enumerate(sizes)]
    alone = [sd.vl_hog_polar(_dev(m[None]), _dev(a[None]), cs, K, variant, directed=bool(directed),
                             bilinear_orientations=bool(bil))[0] for m, a in fields]
    # fields packed with gaps, odd ones stored transposed (column-major: pixel stride h, row stride 1)
    mparts, aparts, descs, pos = [], [], [], 3
    for i, (m, a) in enumerate(fields):
        h, w = m.shape
        tr = i % 2 == 1
        mparts += [np.zeros(3 if i == 0 else 5, np.float32), (m.T if tr else m).ravel()]
        aparts += [np.zeros(3 if i == 0 else 5, np.float32), (a.T if tr else a).ravel()]
        descs.append(HogImageC(w, h, pos, 1 if tr else w, h if tr else 1, 0))
        pos += m.size + 5
    bm, ba = _dev(np.concatenate(mparts)), _dev(np.concatenate(aparts))
    table = (HogImageC * len(descs))(*descs)
    d_table = _dev(np.frombuffer(bytes(table), dtype=np.uint8).copy())
    fb = HogPolarFieldsC(C.c_void_p(bm.data_ptr()), C.c_void_p(ba.data_ptr()), len(fields), HogImageC(), 0, C.c_void_p(d_table.data_ptr()))
    gap, sentinel = 5, -1234.5
    starts, p = [], gap
    for x in alone:
        starts.append(p)
        p += x.numel() + gap
    offsets = torch.tensor(starts, dtype=torch.int64, device="cuda")
    runs = []
    for _ in range(2):
        out = torch.full((p,), sentinel, dtype=torch.float32, device="cuda")
        assert _polar_into(ctx, fb, cs, K, variant, directed, bil, out, offsets) == 0
        runs.append(out.cpu().numpy())
    assert np.array_equal(runs[0], runs[1])
    mask = np.ones(p, dtype=bool)
    for s, x in zip(starts, alone):
        assert np.array_equal(runs[0][s:s + x.numel()], x.cpu().numpy().ravel())
        mask[s:s + x.numel()] = False
    assert np.all(runs[0][mask] == sentinel)
    # one size, NULL offsets: field i at i * dd * hogH * hogW, and the same field among others in a batch
    eq = [smooth_field(97, 131, seed=50 + i) for i in range(6)]
    em, ea = np.stack([f[0] for f in eq]), np.stack([f[1] for f in eq])
    single = [sd.vl_hog_polar(_dev(em[i:i + 1]), _dev(ea[i:i + 1]), cs, K, variant, directed=bool(directed),
                              bilinear_orientations=bool(bil))[0] for i in range(6)]
    dm, da = _dev(em), _dev(ea)
    fb1 = HogPolarFieldsC(C.c_void_p(dm.data_ptr()), C.c_void_p(da.data_ptr()), 6, HogImageC(131, 97, 0, 131, 1, 0), 97 * 131, None)
    per = single[0].numel()
    out = torch.full((6 * per + gap,), sentinel, dtype=torch.float32, device="cuda")
    assert _polar_into(ctx, fb1, cs, K, variant, directed, bil, out, None) == 0
    got = out.cpu().numpy()
    for i in range(6):
        assert np.array_equal(got[i * per:(i + 1) * per], single[i].cpu().numpy().ravel()), i
    assert np.all(got[6 * per:] == sentinel)


def test_vl_hog_polar_of_host_fields(sd):
    """numpy batches and lists of mixed sizes equal the device call field by field."""
    import torch
    sizes = [(120, 160), (97, 131), (200, 150), (64, 64)]
    fields = [smooth_field(h, w, seed=70 + i) for i, (h, w) in enumerate(sizes)]
    for cs, K, variant, directed, bil in ((8, 9, 1, True, False), (6, 4, 0, False, True)):
        kw = dict(directed=directed, bilinear_orientations=bil)
        want = [sd.vl_hog_polar(_dev(m[None]), _dev(a[None]), cs, K, variant, **kw)[0] for m, a in fields]
        got = sd.vl_hog_polar([m for m, _ in fields], [a for _, a in fields], cs, K, variant, **kw)
        assert isinstance(got, list) and len(got) == 4
        for i in range(4):
            assert torch.equal(got[i], want[i]), (cs, K, i)
        m0, a0 = fields[0]
        same = sd.vl_hog_polar(np.stack([m0, m0]), np.stack([a0, a0]), cs, K, variant, **kw)
        assert tuple(same.shape[:1]) == (2,) and torch.equal(same[1], want[0])
        same_list = sd.vl_hog_polar([m0, m0], [a0, a0], cs, K, variant, **kw)
        assert torch.equal(same_list[1], want[0])


def test_vl_hog_polar_invalid_arguments(sd):
    """Every invalid case is SD_ERR_INVALID, queues no kernel and leaves out untouched; shape errors in Python are ValueError."""
    import torch
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogImageC, HogPolarFieldsC
    ctx = sd.default_context()
    lib = _capi.lib()
    mod = torch.zeros(2 * 40 * 48 + 4, dtype=torch.float32, device="cuda")
    ang = torch.zeros(2 * 40 * 48 + 4, dtype=torch.float32, device="cuda")
    sentinel = -77.25
    out = torch.full((1 << 16,), sentinel, dtype=torch.float32, device="cuda")

    def fields(w=48, h=40, off=0, rs=48, ps=1, cst=0, count=2, stride=1920, m=None, a=None, frames=None):
        return HogPolarFieldsC(C.c_void_p(mod.data_ptr() if m is None else m), C.c_void_p(ang.data_ptr() if a is None else a), count,
                               HogImageC(w, h, off, rs, ps, cst), stride, C.c_void_p(frames) if frames else None)

    def table(*descs):
        t = (HogImageC * len(descs))(*descs)
        return torch.from_numpy(np.frombuffer(bytes(t), dtype=np.uint8).copy()).cuda()

    good = HogImageC(48, 40, 0, 48, 1, 0)
    d_bad_stride = table(good, HogImageC(48, 40, 1920, -48, 1, 0))
    d_small = table(good, HogImageC(3, 40, 1920, 48, 1, 0))
    d_bad_off = table(good, HogImageC(48, 40, -1, 48, 1, 0))
    d_two = table(good, HogImageC(40, 40, 1920, 40, 1, 0))
    # (fields, cs, K, variant, directed, bilinear)
    cases = [(fields(m=0), 4, 4, 1, 1, 0), (fields(a=0), 4, 4, 1, 1, 0), (fields(m=mod.data_ptr() + 2), 4, 4, 1, 1, 0),
             (fields(a=ang.data_ptr() + 1), 4, 4, 1, 1, 0), (fields(), 4, 4, 1, 2, 0), (fields(), 4, 4, 1, -1, 0),
             (fields(), 4, 4, 1, 1, 2), (fields(), 4, 4, 1, 1, -1), (fields(rs=-48), 4, 4, 1, 1, 0), (fields(ps=-1), 4, 4, 1, 1, 0),
             (fields(cst=-1), 4, 4, 1, 1, 0), (fields(off=-1), 4, 4, 1, 1, 0), (fields(stride=-1920), 4, 4, 1, 1, 0),
             (fields(w=3), 4, 4, 1, 1, 0), (fields(h=3), 4, 4, 1, 1, 1), (fields(w=4), 11, 4, 1, 1, 0), (fields(), 4, 0, 1, 1, 0),
             (fields(), 4, 17, 1, 1, 1), (fields(), 0, 4, 1, 1, 0), (fields(), 33, 4, 1, 1, 1), (fields(), 4, 4, 2, 1, 0),
             (fields(count=-1), 4, 4, 1, 1, 0), (fields(frames=d_bad_stride.data_ptr()), 4, 4, 1, 1, 0),
             (fields(frames=d_small.data_ptr()), 4, 4, 1, 0, 1), (fields(frames=d_bad_off.data_ptr()), 4, 4, 1, 1, 0),
             (fields(frames=d_two.data_ptr()), 4, 4, 1, 1, 0)]
    torch.cuda.synchronize()
    before = ctx.launches()
    for fb, cs, K, variant, directed, bil in cases:
        assert _polar_into(ctx, fb, cs, K, variant, directed, bil, out, None) == 1, \
            (fb.frame.width, fb.frame.height, fb.frame.offset, cs, K, variant, directed, bil)
    assert lib.sd_hog_dense_polar(ctx.h, None, 4, 4, 1, 1, 0, _capi.ptr(out), None) == 1
    assert lib.sd_hog_dense_polar(ctx.h, C.byref(fields()), 4, 4, 1, 1, 0, None, None) == 1
    assert ctx.launches() == before
    assert torch.all(out == sentinel)
    z = np.zeros((2, 40, 48), np.float32)
    for m, a in ((z.astype(np.float64), z), (z, z[:, :, :47]), (z[0], z[0]), ([z[0]], [z[0], z[0]]), ([z[0]], z),
                 ([z[0].astype(np.uint8)], [z[0]]), ([z[0]], [z[0, :, :40]])):
        with pytest.raises(ValueError):
            sd.vl_hog_polar(m, a, 4, 4)
    with pytest.raises(sd.SdError):
        sd.vl_hog_polar(z[:, :3], z[:, :3], 4, 4)

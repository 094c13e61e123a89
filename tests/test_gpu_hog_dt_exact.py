"""The exact transform on the device (sd_hog_distance_transform_exact, sd_hog_part_placements_mapped and vl_hog_part_detect with
max_displacement=None), against the numpy restatement hog_dt_exact_ref.py.

- Values and placements bit for bit on 1 x 1, 1 x n and n x 1 maps, on lines of up to 32 positions (envelopes in shared
  memory) and longer ones (envelopes in scratch), on many maps of different sizes in one call, on a full bank of 256 planes, with
  tiny w0 (a score reaches across the map) and large asymmetric w1, and with NaN and +-inf scores.
- Two runs are identical; on integer maps of at most 32 cells the result equals sd_hog_distance_transform at R = 32.
- Refusals leave canary-filled outputs untouched.
- vl_hog_part_detect with max_displacement=None equals its composition (device pyramid, correlates, exact transform and
  assembly; numpy detections; parts read from the transform's maps), for a model and its flipped() mirror, and equals the
  bounded route at R = 32 where the part maps fit in 32 cells and every part score is an integer.
- (tests/test_cpp_hog_parts_exact.py: the C++ shell returns the Python result bit for bit.)"""
import ctypes as C

import numpy as np
import pytest
import torch

import hog_detect_ref as DR
import hog_dt_exact_ref as ex
import hog_parts_ref as ref
import synth
from superviseddescent_b200._capi import HogGridsC, HogPartMapC, HogPartModelC, ptr

pytestmark = pytest.mark.gpu

CS, K = 8, 9
DD = 3 * K + 4


def _same(vals, place, maps, d):
    for i in range(maps.shape[0]):
        for k in range(maps.shape[1]):
            D, pl = ex.transform(maps[i, k], d[k])
            assert np.array_equal(vals[i, k].view(np.int32), D.view(np.int32)), (i, k)
            assert np.array_equal(place[i, k], pl), (i, k)


def _deformation(rng, P, kind):
    if kind == "tiny":
        return np.stack([np.full(P, 1e-6), rng.normal(0, 1e-4, P), np.full(P, 2e-6), rng.normal(0, 1e-4, P)], 1).astype(np.float32)
    if kind == "asymmetric":
        return np.stack([rng.uniform(0.005, 0.05, P), rng.choice([-9.0, 6.5], P), rng.uniform(0.005, 0.05, P),
                         rng.choice([7.0, -5.5], P)], 1).astype(np.float32)
    return np.stack([rng.uniform(0.01, 0.3, P), rng.normal(0, 0.2, P), rng.uniform(0.01, 0.3, P), rng.normal(0, 0.2, P)],
                    1).astype(np.float32)


@pytest.mark.parametrize("n,P,h,w,kind", [(4, 2, 1, 1, "random"), (2, 3, 1, 150, "random"), (2, 3, 150, 1, "random"),
                                          (3, 2, 20, 31, "random"), (2, 2, 32, 32, "specials"), (2, 2, 17, 70, "random"),
                                          (2, 3, 45, 300, "random"), (1, 2, 90, 155, "tiny"), (1, 2, 64, 97, "asymmetric"),
                                          (2, 2, 40, 41, "specials")])
def test_transform_matches_restatement(sd, n, P, h, w, kind):
    rng = np.random.default_rng(n * 1000 + h * 10 + w)
    maps = rng.normal(0, 2, (n, P, h, w)).astype(np.float32)
    if kind == "specials":
        flat = maps.reshape(-1)
        idx = rng.choice(flat.size, flat.size // 6, replace=False)
        flat[idx[0::3]] = np.nan
        flat[idx[1::3]] = np.inf
        flat[idx[2::3]] = -np.inf
        maps[0, 0, 5:9, :] = np.nan                               # rows without a candidate
        maps[1, 1, :, 3] = -np.inf                                # a column without a candidate
    d = _deformation(rng, P, kind)
    vals, place = sd.vl_hog_distance_transform(torch.from_numpy(maps), d)
    _same(vals.cpu().numpy(), place.cpu().numpy(), maps, d)


def test_many_maps_of_different_sizes(sd):
    rng = np.random.default_rng(5)
    sizes = [(1, 1), (31, 40), (7, 3), (64, 65), (1, 90), (90, 1), (33, 32), (5, 200)]
    maps = [rng.normal(0, 1, (3, h, w)).astype(np.float32) for h, w in sizes]
    d = _deformation(rng, 3, "random")
    before = sd.default_context().launches()
    vals, place = sd.vl_hog_distance_transform([torch.from_numpy(m) for m in maps], d)
    assert sd.default_context().launches() - before == 2                 # pass X and pass Y
    for m, v, p in zip(maps, vals, place):
        _same(v.cpu().numpy()[None], p.cpu().numpy()[None], m[None], d)


def test_full_bank_of_planes(sd):
    rng = np.random.default_rng(9)
    maps = rng.normal(0, 1, (2, 256, 9, 40)).astype(np.float32)
    d = _deformation(rng, 256, "random")
    vals, place = sd.vl_hog_distance_transform(torch.from_numpy(maps), d)
    vals, place = vals.cpu().numpy(), place.cpu().numpy()
    for k in range(256):
        _same(vals[:, k:k + 1], place[:, k:k + 1], maps[:, k:k + 1], d[k:k + 1])


def test_two_runs_are_identical(sd):
    rng = np.random.default_rng(13)
    maps = torch.from_numpy(rng.normal(0, 1, (3, 4, 70, 90)).astype(np.float32))
    d = _deformation(rng, 4, "asymmetric")
    a = sd.vl_hog_distance_transform(maps, d)
    b = sd.vl_hog_distance_transform(maps, d)
    assert torch.equal(a[0].view(torch.int32), b[0].view(torch.int32)) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("h,w", [(1, 1), (32, 32), (13, 29), (32, 1)])
def test_integer_maps_equal_the_bounded_transform_at_32(sd, h, w):
    rng = np.random.default_rng(h * 64 + w)
    maps = rng.integers(-20, 21, (3, 4, h, w)).astype(np.float32)
    d = np.stack([rng.integers(1, 4, 4), rng.integers(-5, 6, 4), rng.integers(1, 4, 4), rng.integers(-5, 6, 4)], 1).astype(np.float32)
    v0, p0 = sd.vl_hog_distance_transform(torch.from_numpy(maps), d)
    v1, p1 = sd.vl_hog_distance_transform(torch.from_numpy(maps), d, 32)
    assert torch.equal(v0.view(torch.int32), v1.view(torch.int32)) and torch.equal(p0, p1)


def test_refusals_write_nothing(sd):
    lib = sd._capi.lib()
    ctx = sd.default_context()
    canary = -1234.5
    maps = torch.zeros((2, 3, 4, 40), device="cuda")
    out = torch.full((2, 3, 4, 40), canary, device="cuda")
    place = torch.full((2, 3, 4, 40, 2), -77, dtype=torch.int32, device="cuda")
    good = np.full((3, 4), 0.5, np.float32)

    def dt(planes=3, d=good, o=out, pl=place, count=2, features=maps):
        g = HogGridsC()
        g.d_features, g.count, g.width, g.height, g.d_grids = features.data_ptr() if features is not None else None, count, 40, 4, None
        dp = np.ascontiguousarray(d, np.float32)
        return lib.sd_hog_distance_transform_exact(ctx.h, C.byref(g), planes, C.c_void_p(dp.ctypes.data), ptr(o), ptr(pl))

    def with_(i, j, v):
        d = good.copy()
        d[i, j] = v
        return d

    for rc in (dt(d=with_(0, 0, 0.0)), dt(d=with_(1, 2, -1.0)), dt(d=with_(2, 2, 0.0)), dt(d=with_(0, 1, np.inf)),
               dt(d=with_(1, 3, np.nan)), dt(d=with_(2, 0, np.inf)), dt(planes=0), dt(planes=257, d=np.full((257, 4), 0.5)),
               dt(o=None), dt(count=-1), dt(features=None), dt(pl=place.view(-1)[1:]), dt(o=out.view(-1)[1:].view(torch.uint8)[1:])):
        assert rc != 0
    torch.cuda.synchronize()
    assert torch.all(out == canary) and torch.all(place == -77)

    # the mapped placements
    anchors = torch.zeros((2, 3, 2), dtype=torch.int32, device="cuda")
    m = HogPartModelC(2, 3, 4, 4, 2, 2, 0, 0, 0, 0, anchors.data_ptr())
    values = torch.zeros(6 * 8 * 8, device="cuda")
    pmaps = torch.zeros((6 * 8 * 8, 2), dtype=torch.int32, device="cuda")
    table = sd._device_table([HogPartMapC(0, 0, 64, 64, 64, 64, 3, 3, 8, 8, 0, 0, 0)], "cuda:0")
    det = torch.zeros((1, 4, 9), dtype=torch.int32, device="cuda")
    det[0, 0, 5:9] = torch.tensor([1, 0, 2, 2])
    det[0, 1, 5:9] = torch.tensor([0, 3, 0, 0])                  # level 3: not in the table
    count = torch.tensor([1], dtype=torch.int32, device="cuda")
    count2 = torch.tensor([2], dtype=torch.int32, device="cuda")
    out_p = torch.full((1, 4, 3, 7), -99, dtype=torch.int32, device="cuda")

    def pm(cnt=count, pl=pmaps, md=4):
        return lib.sd_hog_part_placements_mapped(ctx.h, ptr(values), ptr(pl), ptr(table), 1, C.byref(m), CS, ptr(det), ptr(cnt), 1, md,
                                                 ptr(out_p))

    for rc in (pm(cnt=count2), pm(pl=None), pm(pl=pmaps.view(-1)[1:]), pm(md=0)):
        assert rc != 0
    torch.cuda.synchronize()
    assert torch.all(out_p == -99)
    assert pm() == 0
    torch.cuda.synchronize()
    assert torch.all(out_p[0, 1:] == -99) and not torch.all(out_p[0, 0] == -99)


# ---- the detector ------------------------------------------------------------------------------------------------------------
def _model(rng, Q=2, P=3, fw=4, fh=5, pfw=3, pfh=2, pad=(1, 2), part_pad=(2, 1), zero_parts=False, integer=False):
    root = rng.normal(0, 0.2, (Q, DD, fh, fw)).astype(np.float32)
    parts = np.zeros((Q, P, DD, pfh, pfw), np.float32) if zero_parts else rng.normal(0, 0.2, (Q, P, DD, pfh, pfw)).astype(np.float32)
    anchors = np.stack([rng.integers(0, 2 * fw - pfw + 1, (Q, P)), rng.integers(0, 2 * fh - pfh + 1, (Q, P))], -1)
    anchors[1, 1] = (-3, -2)                                      # outside near the top-left border
    if integer:
        deformation = np.stack([rng.integers(1, 3, (Q, P)), rng.integers(-3, 4, (Q, P)), rng.integers(1, 3, (Q, P)),
                                rng.integers(-3, 4, (Q, P))], -1).astype(np.float32)
    else:
        deformation = np.stack([rng.uniform(0.001, 0.1, (Q, P)), rng.normal(0, 0.3, (Q, P)), rng.uniform(0.001, 0.1, (Q, P)),
                                rng.normal(0, 0.3, (Q, P))], -1).astype(np.float32)
    bias = rng.normal(0, 0.1, Q).astype(np.float32)
    return root, bias, parts, anchors, deformation, pad, part_pad


def _composition(sd, frames, scales, m, thr, overlap, mc, md):
    """vl_hog_part_detect restated from its steps: the device pyramid, correlates, exact transform and assembly; the numpy
    detections; and each part read from the transform's maps at its anchor."""
    every = list(dict.fromkeys(scales + [2 * s for s in scales]))
    feats, levels = sd.vl_hog_pyramid(frames, every, CS, K)
    q, p = m.num_components, m.num_parts
    maps, pinfo = [], {}
    for i, fr in enumerate(frames):
        for s, sc in enumerate(scales):
            r, pl = every.index(sc), every.index(2 * sc)
            if feats[i][r] is None:
                continue
            root = sd.vl_hog_correlate([feats[i][r]], m.root, K, bias=m.bias, pad=m.pad)[0]
            if root.numel() == 0:
                continue
            D = place = None
            if feats[i][pl] is not None:
                ps = sd.vl_hog_correlate([feats[i][pl]], m.parts.reshape(q * p, DD, *m.parts.shape[3:]), K, pad=m.part_pad)[0]
                if ps.numel():
                    D, place = sd.vl_hog_distance_transform(ps[None], m.deformation.reshape(-1, 4))
                    D, place = D[0], place[0]
            total = sd.vl_hog_part_scores([root], [D], m)[0].cpu().numpy()
            maps.append(DR.ScoreMap(i, s, fr.shape[1], fr.shape[0], *levels[i][r], total))
            pinfo[(i, s)] = {"D": None if D is None else D.cpu().numpy(), "place": None if place is None else place.cpu().numpy(),
                             "frame_w": fr.shape[1], "frame_h": fr.shape[0],
                             "part_level_w": levels[i][pl][0], "part_level_h": levels[i][pl][1]}
    fh, fw = m.root.shape[2:]
    dets, above = DR.detections(maps, len(frames), CS, fw, fh, m.pad[0], m.pad[1], thr, overlap, mc, md)
    pfh, pfw = m.parts.shape[3:]
    parts = [np.stack([ref.placements(rec, pinfo[(i, int(rec[6]))], m.anchors, m.pad, m.part_pad, (pfw, pfh), CS) for rec in d])
             if len(d) else np.zeros((0, p, 7), np.int32) for i, d in enumerate(dets)]
    return dets, above, parts


def _frames():
    sizes = [(120, 160), (97, 131), (64, 72)]
    return [synth.smooth_images(1, h, w, seed=40 + i, sigma=1.0)[0] for i, (h, w) in enumerate(sizes)]


def _rows(d):
    return (np.concatenate([d.boxes, d.scores.view(np.int32)[:, None], d.filter[:, None], d.level[:, None], d.cell], axis=1),
            np.concatenate([d.placement, d.part_scores.view(np.int32)[..., None], d.parts], axis=2))


@pytest.mark.parametrize("mirror", [False, True])
def test_detector_equals_its_composition(sd, mirror):
    rng = np.random.default_rng(11 + mirror)
    frames = _frames()
    m = sd.HogPartModel(*_model(rng), max_displacement=None)
    if mirror:
        m = m.flipped(K)
        assert m.max_displacement is None
    scales = [0.5, 1.0, 0.8]
    thr, overlap, mc, md = -1.0, 0.4, 300, 40
    d = sd.vl_hog_part_detect(frames, scales, m, CS, K, thr, overlap=overlap, max_candidates=mc, max_detections=md)
    dets, above, parts = _composition(sd, frames, scales, m, thr, overlap, mc, md)
    assert np.array_equal(d.above, above)
    rows, prow = _rows(d)
    assert len(rows) > 10
    for i in range(len(frames)):
        sel = d.frame == i
        assert np.array_equal(rows[sel], dets[i]), i
        assert np.array_equal(prow[sel], parts[i]), i
    assert np.any(prow[..., 0] >= 0)


def test_detector_equals_the_bounded_route_on_integer_part_scores(sd):
    """Zero part filters make every part score 0, an integer; with integer weights every operation of both transforms is exact.
    The frames' part levels give part maps of at most 20 x 15 positions, inside R = 32."""
    rng = np.random.default_rng(17)
    frames = _frames()
    args = _model(rng, zero_parts=True, integer=True)
    exact = sd.HogPartModel(*args, max_displacement=None)
    bounded = sd.HogPartModel(*args, max_displacement=32)
    for m0, m1 in ((exact, bounded), (exact.flipped(K), bounded.flipped(K))):
        a = sd.vl_hog_part_detect(frames, [0.5, 0.4], m0, CS, K, -1e30, overlap=1.0, max_candidates=2000, max_detections=500)
        b = sd.vl_hog_part_detect(frames, [0.5, 0.4], m1, CS, K, -1e30, overlap=1.0, max_candidates=2000, max_detections=500)
        ra, pa = _rows(a)
        rb, pb = _rows(b)
        assert len(ra) > 100 and np.array_equal(ra, rb) and np.array_equal(pa, pb)

"""Deformable part models on the device (sd_hog_distance_transform, sd_hog_part_scores, sd_hog_part_placements and
api.vl_hog_part_detect), against the numpy restatement hog_parts_ref.py.

- Transform: values and placements bit for bit, on random maps, on integer scores with integer costs (ties), with +-inf, NaN
  and all-NaN windows, on 1 x 1 maps, maps smaller than R, R = 0 and R = 32, maps of several sizes through a descriptor table,
  and more than 65,535 planes.
- Assembly and placements: bit for bit through the whole vl_hog_part_detect chain, anchors outside the part map included; the
  placements call's output equals the transform's d_place at every anchor.
- The same call twice is identical, and each frame's result is the same alone and in a batch; every refusal writes nothing.
- Planted objects: textured parts shifted by known whole cells are found at their boxes with every part at its planted shift,
  score above the root alone and above the rigid model, and the mirrored model finds the mirrored instances at the mirrored
  root and part boxes.
- (tests/test_cpp_hog_parts.py: the C++ shell returns the Python result bit for bit.)"""
import ctypes as C

import numpy as np
import pytest
import torch

import hog_detect_ref as DR
import hog_parts_ref as ref
import synth
from superviseddescent_b200._capi import HogGridC, HogGridsC, HogPartMapC, HogPartModelC, ptr

pytestmark = pytest.mark.gpu

CS, K = 8, 9
DD = 3 * K + 4


def _check_transform(sd, maps, deformation, R):
    """maps (N, P, h, w) float32 -> bit-exact comparison of values and placements with the restatement, per plane."""
    vals, place = sd.vl_hog_distance_transform(torch.from_numpy(maps), deformation, R)
    vals, place = vals.cpu().numpy(), place.cpu().numpy()
    for i in range(maps.shape[0]):
        for k in range(maps.shape[1]):
            D, pl = ref.transform(maps[i, k], deformation[k], R)
            assert np.array_equal(vals[i, k].view(np.int32), D.view(np.int32)), (i, k)
            assert np.array_equal(place[i, k], pl), (i, k)


@pytest.mark.parametrize("n,P,h,w,R,kind", [(3, 2, 37, 45, 4, "random"), (2, 3, 70, 33, 16, "random"), (2, 2, 40, 41, 3, "integer"),
                                            (1, 4, 9, 64, 32, "random"), (2, 2, 5, 3, 16, "random"), (4, 1, 1, 1, 7, "random"),
                                            (2, 2, 13, 17, 0, "random"), (2, 2, 35, 34, 2, "specials"), (1, 2, 33, 65, 32, "integer")])
def test_transform_matches_restatement(sd, n, P, h, w, R, kind):
    rng = np.random.default_rng(n * 1000 + h * 10 + w + R)
    if kind == "integer":
        maps = rng.integers(-3, 4, (n, P, h, w)).astype(np.float32)
        deformation = rng.integers(0, 3, (P, 4)).astype(np.float32)
        deformation[:, [1, 3]] = rng.integers(-2, 3, (P, 2))
    else:
        maps = rng.normal(0, 2, (n, P, h, w)).astype(np.float32)
        deformation = np.stack([rng.uniform(0, 0.3, P), rng.normal(0, 0.2, P), rng.uniform(0, 0.3, P), rng.normal(0, 0.2, P)], 1)
    if kind == "specials":
        flat = maps.reshape(-1)
        idx = rng.choice(flat.size, flat.size // 6, replace=False)
        flat[idx[0::3]] = np.nan
        flat[idx[1::3]] = np.inf
        flat[idx[2::3]] = -np.inf
        maps[0, 0, 5:14, 3:12] = np.nan                          # windows with no candidate at R = 2
        maps[1, 1, :, 20:] = np.nan
    _check_transform(sd, maps, deformation.astype(np.float32), R)


def test_transform_of_a_table_of_sizes(sd):
    rng = np.random.default_rng(5)
    sizes = [(1, 1), (31, 40), (7, 3), (64, 65)]
    maps = [rng.normal(0, 1, (3, h, w)).astype(np.float32) for h, w in sizes]
    d = np.array([[0.1, 0.0, 0.2, 0.05], [0.3, -0.1, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0]], np.float32)
    vals, place = sd.vl_hog_distance_transform([torch.from_numpy(m) for m in maps], d, 5)
    for m, v, p in zip(maps, vals, place):
        for k in range(3):
            D, pl = ref.transform(m[k], d[k], 5)
            assert np.array_equal(v[k].cpu().numpy().view(np.int32), D.view(np.int32))
            assert np.array_equal(p[k].cpu().numpy(), pl)


def test_transform_past_65535_planes(sd):
    rng = np.random.default_rng(7)
    base = rng.normal(0, 1, (7, 2, 3, 4)).astype(np.float32)
    n = 32776                                                    # 65,552 planes
    maps = base[np.arange(n) % 7]
    d = np.array([[0.2, 0.1, 0.3, -0.1], [0.05, 0.0, 0.05, 0.0]], np.float32)
    before = sd.default_context().launches()
    vals, place = sd.vl_hog_distance_transform(torch.from_numpy(maps), d, 2)
    assert sd.default_context().launches() - before == 1
    vals, place = vals.cpu().numpy(), place.cpu().numpy()
    for b in range(7):
        for k in range(2):
            D, pl = ref.transform(base[b, k], d[k], 2)
            assert np.array_equal(vals[b::7, k].view(np.int32), np.broadcast_to(D.view(np.int32), vals[b::7, k].shape))
            assert np.array_equal(place[b::7, k], np.broadcast_to(pl, place[b::7, k].shape))


def _model(rng, Q=2, P=3, fw=4, fh=5, pfw=3, pfh=2, pad=(1, 2), part_pad=(2, 1), R=3, outside=True):
    root = rng.normal(0, 0.2, (Q, DD, fh, fw)).astype(np.float32)
    parts = rng.normal(0, 0.2, (Q, P, DD, pfh, pfw)).astype(np.float32)
    anchors = np.stack([rng.integers(0, 2 * fw - pfw + 1, (Q, P)), rng.integers(0, 2 * fh - pfh + 1, (Q, P))], -1)
    if outside:
        anchors[0, 0] = (2 * fw + 40, 1)                          # outside the part map everywhere
        anchors[1, 1] = (-3, -2)                                  # outside near the top-left border
    deformation = np.stack([rng.uniform(0.01, 0.2, (Q, P)), rng.normal(0, 0.1, (Q, P)), rng.uniform(0.01, 0.2, (Q, P)),
                            rng.normal(0, 0.1, (Q, P))], -1).astype(np.float32)
    bias = rng.normal(0, 0.1, Q).astype(np.float32)
    return root, bias, parts, anchors, deformation, pad, part_pad, R


def _chain_reference(sd, frames, scales, m, thr, overlap, mc, md):
    """The detector restated: the device pyramid and correlates, then the numpy transform, assembly, detections and parts."""
    every = list(dict.fromkeys(scales + [2 * s for s in scales]))
    feats, levels = sd.vl_hog_pyramid(frames, every, CS, K)
    q, p = m.num_components, m.num_parts
    maps, pinfo = [], {}
    for i, fr in enumerate(frames):
        for s, sc in enumerate(scales):
            r, pl = every.index(sc), every.index(2 * sc)
            if feats[i][r] is None:
                continue
            root = sd.vl_hog_correlate([feats[i][r]], m.root, K, bias=m.bias, pad=m.pad)[0].cpu().numpy()
            if root.size == 0:
                continue
            D = place = None
            if feats[i][pl] is not None:
                ps = sd.vl_hog_correlate([feats[i][pl]], m.parts.reshape(q * p, DD, *m.parts.shape[3:]), K, pad=m.part_pad)[0].cpu().numpy()
                if ps.size:
                    tr = [ref.transform(ps[k], m.deformation.reshape(-1, 4)[k], m.max_displacement) for k in range(q * p)]
                    D = np.stack([t[0] for t in tr])
                    place = np.stack([t[1] for t in tr])
            total = ref.part_scores(root, D, m.anchors, m.pad, m.part_pad)
            maps.append(DR.ScoreMap(i, s, fr.shape[1], fr.shape[0], *levels[i][r], total))
            pinfo[(i, s)] = {"D": D, "place": place, "frame_w": fr.shape[1], "frame_h": fr.shape[0],
                             "part_level_w": levels[i][pl][0], "part_level_h": levels[i][pl][1]}
    fh, fw = m.root.shape[2:]
    dets, above = DR.detections(maps, len(frames), CS, fw, fh, m.pad[0], m.pad[1], thr, overlap, mc, md)
    pfh, pfw = m.parts.shape[3:]
    parts = [np.stack([ref.placements(rec, pinfo[(i, int(rec[6]))], m.anchors, m.pad, m.part_pad, (pfw, pfh), CS) for rec in d])
             if len(d) else np.zeros((0, p, 7), np.int32) for i, d in enumerate(dets)]
    return dets, above, parts


def _frames(rng):
    sizes = [(120, 160), (97, 131), (64, 72)]
    return [synth.smooth_images(1, h, w, seed=40 + i, sigma=1.0)[0] for i, (h, w) in enumerate(sizes)]


def _as_rows(d):
    return np.concatenate([d.boxes, d.scores.view(np.int32)[:, None], d.filter[:, None], d.level[:, None], d.cell], axis=1)


def _parts_rows(d):
    return np.concatenate([d.placement, d.part_scores.view(np.int32)[..., None], d.parts], axis=2)


@pytest.mark.parametrize("R", [0, 3, 32])
def test_detector_matches_restatement(sd, R):
    rng = np.random.default_rng(11 + R)
    frames = _frames(rng)
    m = sd.HogPartModel(*_model(rng, R=R)[:7], max_displacement=R)
    scales = [0.5, 1.0, 0.8]
    thr, overlap, mc, md = -1.0, 0.4, 300, 40
    d = sd.vl_hog_part_detect(frames, scales, m, CS, K, thr, overlap=overlap, max_candidates=mc, max_detections=md)
    dets, above, parts = _chain_reference(sd, frames, scales, m, thr, overlap, mc, md)
    assert np.array_equal(d.above, above)
    rows, prow = _as_rows(d), _parts_rows(d)
    assert len(rows) > 10
    for i in range(len(frames)):
        sel = d.frame == i
        assert np.array_equal(rows[sel], dets[i]), i
        assert np.array_equal(prow[sel], parts[i]), i
    # component 0's part 0 is anchored outside every part map: its totals are -inf and never candidates
    assert np.sum(d.filter == 0) == 0 and np.sum(d.filter == 1) > 0


def test_placements_equal_the_transform_at_the_anchors(sd):
    rng = np.random.default_rng(3)
    frames = _frames(rng)
    m = sd.HogPartModel(*_model(rng, outside=False, R=4)[:7], max_displacement=4)
    d = sd.vl_hog_part_detect(frames, [0.5, 0.7], m, CS, K, -1e30, overlap=1.0, max_candidates=500, max_detections=100)
    every = list(dict.fromkeys([0.5, 0.7, 1.0, 1.4]))
    feats, _ = sd.vl_hog_pyramid(frames, every, CS, K)
    q, p = m.num_components, m.num_parts
    checked = 0
    for k in range(len(d.frame)):
        i, s = int(d.frame[k]), int(d.level[k])
        pl = every.index(2 * [0.5, 0.7][s])
        ps = sd.vl_hog_correlate([feats[i][pl]], m.parts.reshape(q * p, DD, *m.parts.shape[3:]), K, pad=m.part_pad)[0]
        vals, place = sd.vl_hog_distance_transform(ps[None], m.deformation.reshape(-1, 4), 4)
        vals, place = vals[0].cpu().numpy(), place[0].cpu().numpy()
        qq, (x, y) = int(d.filter[k]), d.cell[k]
        for j in range(p):
            u0 = 2 * (x - m.pad[0]) + m.anchors[qq, j, 0] + m.part_pad[0]
            v0 = 2 * (y - m.pad[1]) + m.anchors[qq, j, 1] + m.part_pad[1]
            if 0 <= u0 < vals.shape[2] and 0 <= v0 < vals.shape[1]:
                assert np.array_equal(d.placement[k, j], place[qq * p + j, v0, u0])
                assert d.part_scores[k, j].view(np.int32) == vals[qq * p + j, v0, u0].view(np.int32)
                checked += 1
    assert checked >= 100


def test_deterministic_and_batch_independent(sd):
    rng = np.random.default_rng(21)
    frames = _frames(rng)
    m = sd.HogPartModel(*_model(rng, R=5)[:7], max_displacement=5)
    args = ([0.5, 1.0], m, CS, K, -0.5)
    a = sd.vl_hog_part_detect(frames, *args)
    b = sd.vl_hog_part_detect(frames, *args)
    for f in a._fields:
        assert np.array_equal(getattr(a, f), getattr(b, f)), f
    for i in range(len(frames)):
        alone = sd.vl_hog_part_detect([frames[i]], *args)
        sel = a.frame == i
        assert np.array_equal(_as_rows(alone), _as_rows(a)[sel]) and np.array_equal(_parts_rows(alone), _parts_rows(a)[sel])


def test_refusals_write_nothing(sd):
    lib = sd._capi.lib()
    ctx = sd.default_context()
    canary = -1234.5
    maps = torch.zeros((2, 3, 4, 5), device="cuda")
    out = torch.full((2, 3, 4, 5), canary, device="cuda")
    place = torch.full((2, 3, 4, 5, 2), -77, dtype=torch.int32, device="cuda")
    good = np.full((3, 4), 0.5, np.float32)

    def dt(planes=3, d=good, R=4, o=out, pl=place, count=2, features=maps):
        g = HogGridsC()
        g.d_features, g.count, g.width, g.height, g.d_grids = features.data_ptr() if features is not None else None, count, 5, 4, None
        dp = np.ascontiguousarray(d, np.float32)
        return lib.sd_hog_distance_transform(ctx.h, C.byref(g), planes, C.c_void_p(dp.ctypes.data), R, ptr(o), ptr(pl))

    assert dt() == 0
    torch.cuda.synchronize()
    out.fill_(canary)
    place.fill_(-77)
    bad_def = good.copy()
    bad_def[1, 0] = np.inf
    huge = good.copy()
    huge[2, 2] = 3e38
    for rc in (dt(R=-1), dt(R=33), dt(d=bad_def), dt(d=huge, R=32), dt(planes=0), dt(planes=257, d=np.zeros((257, 4))),
               dt(o=None), dt(count=-1), dt(features=None), dt(pl=place.view(-1)[1:])):
        assert rc != 0
    torch.cuda.synchronize()
    assert torch.all(out == canary) and torch.all(place == -77)

    # the assembly and the placements
    anchors = torch.zeros((2, 3, 2), dtype=torch.int32, device="cuda")

    def model(Q=2, P=3, fw=4, fh=4, pw=2, ph=2, pad=(0, 0), ppad=(0, 0), a=anchors):
        return HogPartModelC(Q, P, fw, fh, pw, ph, pad[0], pad[1], ppad[0], ppad[1], a.data_ptr() if a is not None else None)

    root = torch.zeros(2 * 3 * 3, device="cuda")
    parts = torch.zeros(6 * 8 * 8, device="cuda")
    total = torch.full((2 * 3 * 3,), canary, device="cuda")
    row = HogPartMapC(0, 0, 64, 64, 64, 64, 3, 3, 8, 8, 0, 0, 0)
    table = sd._device_table([row], "cuda:0")
    dup = sd._device_table([row, row], "cuda:0")
    neg = sd._device_table([HogPartMapC(0, 0, 64, 64, 64, 64, 3, -1, 8, 8, 0, 0, 0)], "cuda:0")
    wide = sd._device_table([HogPartMapC(0, 0, 1 << 30, 64, 1, 64, 3, 3, 8, 8, 0, 0, 0)], "cuda:0")   # part boxes past int32

    def ps(m, t=table, n=1):
        return lib.sd_hog_part_scores(ctx.h, ptr(root), ptr(parts), ptr(t), n, C.byref(m), ptr(total))

    for rc in (ps(model(P=0)), ps(model(P=33)), ps(model(Q=86)), ps(model(pw=33)), ps(model(pad=(4, 0))), ps(model(ppad=(0, 2))),
               ps(model(a=None)), ps(model(), n=-1), ps(model(), t=neg)):
        assert rc != 0
    torch.cuda.synchronize()
    assert torch.all(total == canary)

    det = torch.zeros((1, 4, 9), dtype=torch.int32, device="cuda")
    det[0, 0, 5:9] = torch.tensor([1, 0, 2, 2])                  # filter 1, level 0, cell (2, 2)
    det[0, 1, 5:9] = torch.tensor([0, 3, 0, 0])                  # level 3: not in the table
    count = torch.tensor([1], dtype=torch.int32, device="cuda")
    count2 = torch.tensor([2], dtype=torch.int32, device="cuda")
    out_p = torch.full((1, 4, 3, 7), -99, dtype=torch.int32, device="cuda")
    d6 = np.full((6, 4), 0.1, np.float32)

    def pp(m=None, t=table, n=1, d=d6, R=3, cnt=count, md=4):
        m = m or model()
        dp = np.ascontiguousarray(d, np.float32)
        return lib.sd_hog_part_placements(ctx.h, ptr(parts), ptr(t), n, C.byref(m), C.c_void_p(dp.ctypes.data), R, CS, ptr(det),
                                          ptr(cnt), 1, md, ptr(out_p))

    for rc in (pp(t=dup, n=2), pp(cnt=count2), pp(R=33), pp(d=np.full((6, 4), np.nan)), pp(m=model(P=0)), pp(md=0), pp(t=neg),
               pp(t=wide)):
        assert rc != 0
    torch.cuda.synchronize()
    assert torch.all(out_p == -99)
    assert pp() == 0                                             # the valid call writes slot 0 only
    torch.cuda.synchronize()
    assert torch.all(out_p[0, 1:] == -99) and not torch.all(out_p[0, 0] == -99)


# ---- planted objects ---------------------------------------------------------------------------------------------------------
FW = FH = 6                  # root cells at the root level (scale 0.5): 12 x 12 part cells, 96 x 96 px
PS = 4                       # part side, part-level cells
ANCHORS = [(1, 1), (7, 1), (1, 7), (7, 7)]


def _template(rng):
    """P textured 32 x 32 patches of smooth noise: gradients at generic angles, so that the mirrored features are the flipped
    features (an edge at exactly 90 degrees would tie between two bins the same way in the mirror)."""
    return [synth.smooth_images(1, PS * CS, PS * CS, seed=int(rng.integers(1 << 30)), sigma=2.0)[0] for _ in ANCHORS]


def _draw(frame, x, y, patches, shifts):
    frame[y:y + 96, x:x + 96] = 110
    for (ax, ay), (sx, sy), t in zip(ANCHORS, shifts, patches):
        px, py = x + (ax + sx) * CS, y + (ay + sy) * CS
        frame[py:py + PS * CS, px:px + PS * CS] = t


def _planted(sd, seed=0):
    rng = np.random.default_rng(seed)
    patches = _template(rng)
    tmpl = np.full((96, 96), 110.0)
    _draw(tmpl, 0, 0, patches, [(0, 0)] * 4)
    tmpl = tmpl.astype(np.uint8)
    # the model from the HOG of the unshifted template: the root at half resolution, the parts at full resolution
    big = np.full((96 + 32, 96 + 32), 110, np.uint8)             # a margin so that border cells are normalised as in a frame
    big[16:112, 16:112] = tmpl
    full = sd.hog_dense([big], CS, K)[0].cpu().numpy()[:, 2:14, 2:14]
    half = sd.vl_hog_pyramid([big], [0.5], CS, K)[0][0][0].cpu().numpy()[:, 1:7, 1:7]
    root = (half - half.mean())[None]
    parts = np.stack([full[:, ay:ay + PS, ax:ax + PS] - full[:, ay:ay + PS, ax:ax + PS].mean() for ax, ay in ANCHORS])[None]
    deformation = np.tile(np.array([0.02, 0.0, 0.02, 0.0], np.float32), (1, 4, 1))
    model = sd.HogPartModel(root, [0.0], parts, np.array(ANCHORS)[None], deformation, max_displacement=2)
    # frames of 320 x 240 px (multiples of 2 * cell size), two instances each with known shifts
    frames, truth = [], []
    for f in range(3):
        fr = np.full((240, 320), 110.0)
        inst = []
        for x, y in [(32, 48), (176, 112)][: 1 + f % 2]:
            shifts = [tuple(int(v) for v in rng.integers(-1, 2, 2)) for _ in ANCHORS]
            _draw(fr, x, y, patches, shifts)
            inst.append((x, y, shifts))
        frames.append(fr.astype(np.uint8))
        truth.append(inst)
    return model, frames, truth


def _iou(a, b):
    ix = max(0, min(a[0] + a[2], b[0] + b[2]) - max(a[0], b[0]))
    iy = max(0, min(a[1] + a[3], b[1] + b[3]) - max(a[1], b[1]))
    return ix * iy / (a[2] * a[3] + b[2] * b[3] - ix * iy)


def test_planted_parts_are_found_at_their_shifts(sd):
    model, frames, truth = _planted(sd)
    d = sd.vl_hog_part_detect(frames, [0.5], model, CS, K, 0.0, overlap=0.3)
    rigid = sd.HogPartModel(model.root, model.bias, model.parts, model.anchors, model.deformation, max_displacement=0)
    dr = sd.vl_hog_part_detect(frames, [0.5], rigid, CS, K, -1e30, overlap=1.0, max_candidates=8192, max_detections=8192)
    found = 0
    for f, inst in enumerate(truth):
        sel = np.nonzero(d.frame == f)[0]
        for x, y, shifts in inst:
            best = max(sel, key=lambda k: _iou(d.boxes[k], (x, y, 96, 96)))
            assert _iou(d.boxes[best], (x, y, 96, 96)) >= 0.9
            cx, cy = d.cell[best]
            for j, ((ax, ay), (sx, sy)) in enumerate(zip(ANCHORS, shifts)):
                assert tuple(d.placement[best, j]) == (2 * cx + ax + sx, 2 * cy + ay + sy), (f, j)
                assert _iou(d.parts[best, j], (x + (ax + sx) * CS, y + (ay + sy) * CS, PS * CS, PS * CS)) >= 0.9
            # above the root filter alone, and above the rigid model wherever a part is shifted
            root = sd.vl_hog_correlate(sd.vl_hog_pyramid([frames[f]], [0.5], CS, K)[0][0], model.root, K)[0][0].cpu().numpy()
            assert d.scores[best] > root[cy, cx]
            k = np.nonzero((dr.frame == f) & (dr.cell[:, 0] == cx) & (dr.cell[:, 1] == cy))[0]
            assert len(k) == 1 and d.scores[best] >= dr.scores[k[0]]
            if any(s != (0, 0) for s in shifts):
                assert d.scores[best] > dr.scores[k[0]]
            found += 1
    assert found == 4

    # the mirrored model finds the mirrored frames within the correlate's error bar
    mirrored = model.flipped(K)
    dm = sd.vl_hog_part_detect([np.ascontiguousarray(fr[:, ::-1]) for fr in frames], [0.5], mirrored, CS, K, 0.0, overlap=0.3)
    for f, inst in enumerate(truth):
        for x, y, shifts in inst:
            k0 = max(np.nonzero(d.frame == f)[0], key=lambda k: _iou(d.boxes[k], (x, y, 96, 96)))
            mine = np.nonzero(dm.frame == f)[0]
            k1 = max(mine, key=lambda k: _iou(dm.boxes[k], (320 - x - 96, y, 96, 96)))
            b0, b1 = d.boxes[k0], dm.boxes[k1]
            assert (b1[0], b1[1], b1[2], b1[3]) == (320 - b0[0] - b0[2], b0[1], b0[2], b0[3])
            # the patches' top and bottom edges against the flat ground have gradients at exactly 90 degrees, which tie between
            # two bins the same way in the mirror: there the mirrored features differ from the flipped ones by whole votes
            assert abs(float(dm.scores[k1]) - float(d.scores[k0])) <= 0.1 * abs(float(d.scores[k0]))
            for j in range(4):
                p0, p1 = d.parts[k0, j], dm.parts[k1, j]
                assert (p1[0], p1[1]) == (320 - p0[0] - p0[2], p0[1])

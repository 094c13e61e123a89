"""Detections from HOG filter scores on the device (sd_hog_detections, api.vl_hog_detect).

- On random score maps -- several frames, maps of different sizes (empty ones included), frames without maps, Q = 1, 2 and 9,
  scores quantised to a few values so that the tie-break decides, +-0, +-inf and NaN, frames above max_candidates and frames that
  reach max_detections, overlap 0 and 1 -- every field and count equals the numpy restatement (hog_detect_ref.py) bit for bit.
- The same call twice is identical; each frame's result is the same alone and mixed into a larger batch; slots past the count
  keep their canaries.
- Every refusal is SD_ERR_INVALID and writes nothing.
- A textured patch planted cell-aligned in flat frames is the top detection of vl_hog_detect, exactly at its box, and its mirror
  is found by the mirrored filter in the same call.
- The HOG of a golden face, used as a filter, finds that face; its box goes straight into detect_faces.
- (tests/test_cpp_hog_detect.py: the C++ shell returns the Python result bit for bit.)"""
import numpy as np
import pytest
import torch

import hog_detect_ref as R
import synth
from superviseddescent_b200._capi import HogScoreMapC

pytestmark = pytest.mark.gpu

CANARY = -0x2A2A2A2B


def _pack_maps(maps, Q, rng):
    """ScoreMaps -> (device scores with gaps between maps, device table, number of maps)."""
    parts, descs, pos = [], [], 0
    for m in maps:
        gap = int(rng.integers(0, 5))
        parts.append(np.full(gap, 99.0, np.float32))           # never read: a candidate if it were
        pos += gap
        s = np.asarray(m.scores, np.float32).ravel()
        h, w = m.scores.shape[1], m.scores.shape[2]
        descs.append(HogScoreMapC(m.frame, m.level, m.frame_w, m.frame_h, m.level_w, m.level_h, w, h, pos))
        parts.append(s.ravel())
        pos += s.size
    parts.append(np.full(3, 99.0, np.float32))
    scores = torch.from_numpy(np.concatenate(parts)).cuda()
    table = (HogScoreMapC * max(len(descs), 1))(*descs)
    d_table = torch.from_numpy(np.frombuffer(bytes(table), np.uint8).copy()).cuda()
    return scores, d_table, len(descs)


def _call(scores, d_table, n_maps, F, Q, cell, fw, fh, px, py, thr, overlap, mc, md, above=True):
    """-> (rc, out (F, md, 9) int32, count (F,), above (F,)), outputs pre-filled with canaries."""
    from superviseddescent_b200 import _capi, api
    ctx = api.default_context()
    out = torch.full((max(F, 1), max(md, 1), R.FIELDS), CANARY, dtype=torch.int32, device="cuda")
    cnt = torch.full((max(F, 1),), CANARY, dtype=torch.int32, device="cuda")
    ab = torch.full((max(F, 1),), CANARY, dtype=torch.int64, device="cuda")
    rc = _capi.lib().sd_hog_detections(ctx.h, _capi.ptr(scores), _capi.ptr(d_table), n_maps, F, Q, cell, fw, fh, px, py, float(thr),
                                       float(overlap), mc, md, _capi.ptr(out), _capi.ptr(cnt), _capi.ptr(ab if above else None))
    torch.cuda.synchronize()
    return rc, out.cpu().numpy(), cnt.cpu().numpy(), ab.cpu().numpy()


def _random_maps(rng, F, Q, n_maps, quantised, specials, empty_frames=(), big=None):
    maps = []
    frames = [f for f in range(F) if f not in empty_frames]
    for i in range(n_maps):
        f = frames[int(rng.integers(0, len(frames)))]
        W, H = int(rng.integers(40, 1400)), int(rng.integers(40, 900))
        s = float(rng.uniform(0.1, 2.0))
        lw, lh = max(1, int(W * s + 0.5)), max(1, int(H * s + 0.5))
        h, w = (0, int(rng.integers(0, 9))) if i % 7 == 3 else (int(rng.integers(1, 40)), int(rng.integers(1, 50)))
        if big is not None and i == 0:
            f, h, w = big
        if quantised:
            v = rng.integers(-3, 4, (Q, h, w)).astype(np.float32) * np.float32(0.5)
        else:
            v = rng.normal(0, 1, (Q, h, w)).astype(np.float32)
        if specials and v.size:
            flat = v.reshape(-1)
            k = rng.integers(0, flat.size, 12)
            flat[k] = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, np.nan, -0.0, 0.0, np.inf, -0.0, np.nan, 0.0], np.float32)
        maps.append(R.ScoreMap(f, i % 5, W, H, lw, lh, v))
    return maps


def _check_against_oracle(maps, F, Q, cell, fw, fh, px, py, thr, overlap, mc, md, seed, label):
    rng = np.random.default_rng(seed)
    scores, d_table, n = _pack_maps(maps, Q, rng)
    rc, out, cnt, ab = _call(scores, d_table, n, F, Q, cell, fw, fh, px, py, thr, overlap, mc, md)
    assert rc == 0
    ref, ref_above = R.detections(maps, F, cell, fw, fh, px, py, np.float32(thr), overlap, mc, md)
    assert np.array_equal(ab, ref_above), (label, ab, ref_above)
    for f in range(F):
        k = ref[f].shape[0]
        assert cnt[f] == k, (label, f, cnt[f], k)
        assert np.array_equal(out[f, :k], ref[f]), (label, f)
        assert (out[f, k:] == CANARY).all(), (label, f)
    capped = int((ref_above > mc).sum())
    full = sum(int(cnt[f] == md) for f in range(F))
    print(f"{label}: {n} maps, above {ref_above.tolist()}, kept {cnt.tolist()}, {capped} frames above max_candidates, "
          f"{full} at max_detections")
    return scores, d_table, n, out, cnt, ab


CASES = [
    # label, F, Q, n_maps, quantised, specials, empty frames, cell, (fw, fh), (px, py), threshold, overlap, max_c, max_det, big map
    ("Q2 ties capped", 5, 2, 14, True, True, (2,), 8, (6, 6), (2, 3), 0.2, 0.5, 64, 8, None),
    ("Q1 overlap 0", 3, 1, 9, True, True, (), 4, (3, 5), (0, 4), -0.6, 0.0, 4096, 256, None),
    ("Q9 overlap 1", 4, 9, 10, True, True, (0,), 6, (2, 2), (1, 0), 0.7, 1.0, 300, 300, None),
    ("Q1 continuous", 3, 1, 12, False, False, (), 8, (6, 6), (5, 5), 0.5, 0.3, 100, 40, None),
    ("Q2 over the limit", 3, 2, 8, True, True, (), 8, (4, 4), (0, 0), -np.inf, 0.4, 8192, 2000, (1, 90, 80)),
    ("Q1 -inf threshold ties", 2, 1, 6, True, True, (), 5, (1, 1), (0, 0), -np.inf, 0.5, 8192, 8192, (0, 100, 100)),
    ("Q9 one candidate", 2, 9, 5, False, True, (1,), 8, (6, 6), (0, 0), 3.5, 0.5, 1, 1, None),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_detections_match_oracle(sd, case):
    label, F, Q, n_maps, quant, spec, empty, cell, (fw, fh), (px, py), thr, ov, mc, md, big = CASES[case]
    rng = np.random.default_rng(100 + case)
    maps = _random_maps(rng, F, Q, n_maps, quant, spec, empty, big)
    _check_against_oracle(maps, F, Q, cell, fw, fh, px, py, thr, ov, mc, md, case, label)


def test_deterministic_and_batch_independent(sd):
    rng = np.random.default_rng(7)
    F, Q = 4, 2
    args = (8, 6, 6, 2, 3, 0.2, 0.5, 64, 8)
    maps = _random_maps(rng, F, Q, 16, True, True)
    scores, d_table, n, out, cnt, ab = _check_against_oracle(maps, F, Q, *args, seed=1, label="batch")
    _, out2, cnt2, ab2 = _call(scores, d_table, n, F, Q, *args)
    assert np.array_equal(out, out2) and np.array_equal(cnt, cnt2) and np.array_equal(ab, ab2)
    others = _random_maps(np.random.default_rng(8), 3, Q, 9, True, True)
    for f in range(F):
        mine = [m._replace(frame=0) for m in maps if m.frame == f]
        rc, o1, c1, a1 = _call(*_pack_maps(mine, Q, rng), 1, Q, *args) if mine else (0, None, np.zeros(1), np.zeros(1))
        assert rc == 0 and c1[0] == cnt[f] and a1[0] == ab[f]
        if mine:
            assert np.array_equal(o1[0, :cnt[f]], out[f, :cnt[f]])
        # mixed into a larger batch as frame 2, in the same relative order
        mixed = []
        for i, m in enumerate(others):
            mixed.append(m._replace(frame={0: 0, 1: 1, 2: 3}[m.frame]))
            if i < len(mine):
                mixed.append(mine[i]._replace(frame=2))
        mixed += [m._replace(frame=2) for m in mine[len(others):]]
        rc, o2, c2, a2 = _call(*_pack_maps(mixed, Q, rng), 4, Q, *args)
        assert rc == 0 and c2[2] == cnt[f] and a2[2] == ab[f]
        assert np.array_equal(o2[2, :cnt[f]], out[f, :cnt[f]])


def test_refusals_write_nothing(sd):
    from superviseddescent_b200 import _capi, api
    rng = np.random.default_rng(3)
    F, Q = 2, 2
    good = dict(F=F, Q=Q, cell=8, fw=6, fh=6, px=0, py=0, thr=0.0, overlap=0.5, mc=64, md=8)
    maps = _random_maps(rng, F, Q, 4, True, False)
    scores, d_table, n = _pack_maps(maps, Q, rng)
    rc, *_ = _call(scores, d_table, n, **good)
    assert rc == 0

    def bad(**kw):
        a = dict(good)
        a.update(kw)
        return a

    for kw in [dict(F=0), dict(mc=0), dict(mc=8193), dict(md=0), dict(md=65), dict(overlap=-0.1), dict(overlap=1.5),
               dict(overlap=float("nan")), dict(thr=float("nan")), dict(cell=0), dict(cell=33), dict(fw=0), dict(fh=33),
               dict(px=6), dict(py=-1), dict(Q=0), dict(Q=257)]:
        rc, out, cnt, ab = _call(scores, d_table, n, **bad(**kw))
        assert rc == 1, kw
        assert (out == CANARY).all() and (cnt == CANARY).all() and (ab == CANARY).all(), kw
        print("refused:", kw, _capi.lib().sd_last_error(api.default_context().h).decode())
    # pointers: null, unaligned
    ctx = api.default_context()
    out = torch.full((F, 8, R.FIELDS), CANARY, dtype=torch.int32, device="cuda")
    cnt = torch.full((F,), CANARY, dtype=torch.int32, device="cuda")
    ab = torch.full((F + 1,), CANARY, dtype=torch.int64, device="cuda")
    p = _capi.ptr
    L = _capi.lib()
    for s_, t_, o_, c_, a_ in [(None, d_table, out, cnt, ab), (scores, None, out, cnt, ab), (scores, d_table, None, cnt, ab),
                               (scores, d_table, out, None, ab), (scores.data_ptr() + 2, d_table, out, cnt, ab),
                               (scores, d_table.data_ptr() + 4, out, cnt, ab), (scores, d_table, out.data_ptr() + 1, cnt, ab),
                               (scores, d_table, out, cnt.data_ptr() + 2, ab), (scores, d_table, out, cnt, ab.data_ptr() + 4)]:
        rc = L.sd_hog_detections(ctx.h, p(s_), p(t_), n, F, Q, 8, 6, 6, 0, 0, 0.0, 0.5, 64, 8, p(o_), p(c_), p(a_))
        torch.cuda.synchronize()
        assert rc == 1
        assert (out == CANARY).all() and (cnt == CANARY).all() and (ab == CANARY).all()
    # bad map descriptors
    for field, value in [("frame", F), ("frame", -1), ("offset", -1), ("frame_w", 0), ("frame_h", 0), ("level_w", 0),
                         ("level_h", 0), ("width", -1), ("height", -2), ("level_w", 1)]:
        bad_maps = [R.ScoreMap(0, 0, 640, 480, 320, 240, np.zeros((Q, 3, 4), np.float32))]
        sc, tb, nn = _pack_maps(bad_maps, Q, rng)
        raw = bytearray(tb.cpu().numpy().tobytes())
        d = HogScoreMapC.from_buffer(raw)
        setattr(d, field, value)
        if field == "level_w" and value == 1:         # a frame 2^30 px wide at a 1 px level: boxes beyond int32
            d.frame_w = 2 ** 30
        tb = torch.frombuffer(raw, dtype=torch.uint8).cuda()
        rc, out2, cnt2, ab2 = _call(sc, tb, nn, **good)
        assert rc == 1, (field, value)
        assert (out2 == CANARY).all() and (cnt2 == CANARY).all() and (ab2 == CANARY).all()
    # no maps: zero counts
    rc, out2, cnt2, ab2 = _call(None, None, 0, **good)
    assert rc == 0 and (cnt2 == 0).all() and (ab2 == 0).all() and (out2 == CANARY).all()


def _plant_frames(rng, n, H=240, W=320, cell=8, side=5):
    """Flat frames with a textured patch of side x side cells and its mirror, cell-aligned -> (frames, patch boxes, mirror boxes)."""
    P = side * cell
    # smooth noise: gradients at generic angles.  Blocks would have edges at exactly 90 degrees, which lie between two of the 18
    # directed bins at K = 9; the nearest-bin tie then goes the same way in the mirror, and the mirrored filter would not match.
    patch = synth.smooth_images(1, P, P, seed=int(rng.integers(1 << 30)), sigma=2.0)[0]
    frames, plant, mirror = [], [], []
    for i in range(n):
        fr = np.full((H, W), 128, np.uint8)
        x, y = cell * int(rng.integers(1, 12)), cell * int(rng.integers(1, (H - P) // cell - 1))
        xm = x + P + cell * int(rng.integers(2, (W - x - 2 * P) // cell))
        ym = cell * int(rng.integers(1, (H - P) // cell - 1))
        fr[y:y + P, x:x + P] = patch
        fr[ym:ym + P, xm:xm + P] = patch[:, ::-1]
        frames.append(fr)
        plant.append((x, y, P, P))
        mirror.append((xm, ym, P, P))
    return frames, plant, mirror


def test_planted_template(sd):
    rng = np.random.default_rng(11)
    cell, K, side = 8, 9, 5
    frames, plant, mirror = _plant_frames(rng, 4, cell=cell, side=side)
    feats = sd.hog_dense(frames[:1], cell, K, 1)[0]
    x, y = plant[0][0] // cell, plant[0][1] // cell
    f = feats[:, y:y + side, x:x + side]
    f = (f - f.mean()).contiguous()
    filt = torch.stack([f, sd.vl_hog_flip([f], K, 1)[0]])
    scales = [1.25, 1.0, 0.8, 0.6]
    d = sd.vl_hog_detect(frames, scales, filt, cell, K, threshold=0.0, overlap=0.5, max_candidates=4096, max_detections=64)
    allk = sd.vl_hog_detect(frames, scales, filt, cell, K, threshold=0.0, overlap=1.0, max_candidates=8192, max_detections=8192)
    for i in range(len(frames)):
        mine = d.frame == i
        b, s, q, lv = d.boxes[mine], d.scores[mine], d.filter[mine], d.level[mine]
        assert tuple(b[0]) == plant[i] and q[0] == 0 and lv[0] == 1, (i, b[:3], q[:3], lv[:3])
        hit = [k for k in range(len(b)) if tuple(b[k]) == mirror[i] and q[k] == 1]
        a = allk.frame == i
        others = [allk.scores[a][k] for k in range(int(a.sum())) if tuple(allk.boxes[a][k]) not in (plant[i], mirror[i])]
        margin = float(s[0] - max(others))
        print(f"frame {i}: top {s[0]:.4f}, mirror by the mirrored filter {s[hit[0]] if hit else float('nan'):.4f}, margin over any "
              f"other box {margin:.4f}, {int(d.above[i])} candidates")
        assert hit, (i, mirror[i], b[:5], q[:5])
        assert margin > 0


def test_face_filter_chains_to_landmarks(sd, golden):
    import cv2
    gray = np.ascontiguousarray(golden.examples["gray0"])
    bx, by, bw, bh = (int(v) for v in golden.examples["boxes"][0])
    crop = cv2.resize(gray[by:by + bh, bx:bx + bw], (128, 128), interpolation=cv2.INTER_LINEAR)
    cell, K = 8, 9
    f = sd.hog_dense(crop[None], cell, K, 1)[0]
    f = (f - f.mean()).contiguous()
    s0 = 128.0 / bw
    scales = [s0 * k for k in (0.7, 0.85, 1.0, 1.2, 1.4)]
    d = sd.vl_hog_detect([gray], scales, f[None], cell, K, threshold=0.0, overlap=0.3, max_detections=16)
    assert d.boxes.shape[0] >= 1
    x, y, w, h = (int(v) for v in d.boxes[0])
    iw = max(0, min(x + w, bx + bw) - max(x, bx))
    ih = max(0, min(y + h, by + bh) - max(y, by))
    iou = iw * ih / (w * h + bw * bh - iw * ih)
    print(f"top detection {d.boxes[0].tolist()} at scale {scales[d.level[0]]:.4f}, score {d.scores[0]:.4f}; golden box "
          f"{[bx, by, bw, bh]}; IoU {iou:.3f}")
    assert iou >= 0.5
    model = sd.load_detection_model(golden.model_path)
    lm = model.detect_faces([gray], d.frame[:1], boxes=d.boxes[:1])
    assert lm.shape == (1, 2 * model.num_landmarks) and np.isfinite(lm).all()

"""Detection, training and part models on float frames (float_frames=True of vl_hog_detect, train_hog_filter and
vl_hog_part_detect).

- Each call equals its own composition over vl_hog_pyramid(multichannel=True, float_frames=True): detect with the correlate and
  the numpy detection rule; training with the trainer's rule restated on the public primitives (hog_train_ref.train_rule); part
  detect with the correlates, the exact transform, the assembly, the numpy detections and the placements.
- Float frames holding the integer values of 8-bit frames give the 8-bit colour route's detections, filter, bias and part
  placements where both resize rules are exact: the level of the frame's own size, and 2x upscales of multiples of 16.
- A filter trained on float frames in [0, 1] finds every held-out planted object.
- The Python calls refuse float32 frames without float_frames, float_frames without multichannel, and uint8 frames with it;
  sd_hog_train_filter_float refuses other dtypes and unaligned frames before writing anything."""
import numpy as np
import pytest
import torch

import hog_detect_ref as DR
import hog_train_ref as T
import test_gpu_hog_dt_exact as dtx

pytestmark = pytest.mark.gpu

CELL, K, SIDE = 8, 9, 6
DD = 3 * K + 4


class _FloatRoute:
    """The api with vl_hog_pyramid and vl_hog_detect on float frames, for restatements written against those two calls."""

    def __init__(self, sd):
        self._sd = sd

    def __getattr__(self, name):
        return getattr(self._sd, name)

    def vl_hog_pyramid(self, *a, **kw):
        return self._sd.vl_hog_pyramid(*a, multichannel=True, float_frames=True, **kw)

    def vl_hog_detect(self, *a, **kw):
        return self._sd.vl_hog_detect(*a, multichannel=True, float_frames=True, **kw)


def _colour(planes, seed):
    """(H, W) uint8 planes -> float32 (H, W, 3) frames in [0, 1] whose channels differ: the plane, its negative with a
    gradient, and a noisy mix."""
    rng = np.random.default_rng(seed)
    out = []
    for p in planes:
        g = p.astype(np.float32) / np.float32(255)
        ramp = np.linspace(0, 0.2, p.shape[1], dtype=np.float32)[None, :]
        mix = 0.5 * g + rng.uniform(0, 0.05, p.shape).astype(np.float32)
        out.append(np.ascontiguousarray(np.stack([g, 1 - g + ramp, mix], -1).astype(np.float32)))
    return out


def _rows(d):
    return np.concatenate([d.boxes, d.scores.view(np.int32)[:, None], d.filter[:, None], d.level[:, None], d.cell], axis=1)


def _same_detections(a, b):
    for x, y in zip(a, b):
        assert np.array_equal(np.asarray(x), np.asarray(y))


def test_detect_equals_its_composition(sd):
    rng = np.random.default_rng(1)
    planes, _ = T.planted_frames(23, 4, 200, 150, sides=(40, 80))
    frames = _colour([planes[0], planes[1], planes[2][:97, :131], planes[3][:120]], 2)
    filters = rng.normal(0, 0.2, (2, DD, 4, 5)).astype(np.float32)
    bias, pad, scales = [0.1, -0.2], (1, 2), [1.0, 0.8, 0.5, 1.7]
    thr, overlap, mc, md = -0.5, 0.4, 500, 40
    d = sd.vl_hog_detect(frames, scales, filters, CELL, K, thr, bias=bias, pad=pad, overlap=overlap, max_candidates=mc,
                         max_detections=md, multichannel=True, float_frames=True)
    feats, levels = sd.vl_hog_pyramid(frames, scales, CELL, K, multichannel=True, float_frames=True)
    maps = []
    for i, fr in enumerate(frames):
        for s in range(len(scales)):
            if feats[i][s] is None:
                continue
            sc = sd.vl_hog_correlate([feats[i][s]], filters, K, bias=bias, pad=pad)[0].cpu().numpy()
            maps.append(DR.ScoreMap(i, s, fr.shape[1], fr.shape[0], *levels[i][s], sc))
    dets, above = DR.detections(maps, len(frames), CELL, 5, 4, pad[0], pad[1], thr, overlap, mc, md)
    assert np.array_equal(d.above, above)
    rows = _rows(d)
    assert len(rows) > 20
    for i in range(len(frames)):
        assert np.array_equal(rows[d.frame == i], dets[i]), i


def test_trainer_equals_its_composition(sd):
    planes, boxes = T.planted_frames(78, 10, 240, 180, sides=(48, 96), distractors=5)
    frames = _colour(planes, 3)
    scales = T.detector_scales(240, 180, CELL, 5)
    box_frame = np.arange(8)                                      # frames 8 and 9 are pure negative frames
    kw = dict(lam=0.1, flip_positives=True, rounds=3, negatives_per_frame=16, mine_overlap=0.5, max_negatives=40,
              negative_overlap=0.3, positive_overlap=0.6, max_iterations=50)
    hf = sd.train_hog_filter(frames, box_frame, boxes[:8], scales, (5, 5), CELL, K, multichannel=True, float_frames=True, **kw)
    filt, bias, neg, reps = T.train_rule(_FloatRoute(sd), frames, box_frame, boxes[:8], scales, (5, 5), CELL, K, **kw)
    assert np.array_equal(hf.negatives, neg)
    got = [{k: r[k] for k in T.COUNTS + ("solve",)} for r in hf.report]
    assert got[:len(reps)] == reps
    assert np.array_equal(hf.filter.cpu().numpy().ravel().view(np.uint32), filt.view(np.uint32))
    assert np.float32(hf.bias) == bias
    assert sum(r["added"] for r in reps) > 0


@pytest.mark.parametrize("mirror", [False, True])
def test_part_detect_equals_its_composition(sd, mirror):
    rng = np.random.default_rng(31 + mirror)
    frames = _colour(dtx._frames(), 4)
    m = sd.HogPartModel(*dtx._model(rng), max_displacement=None)
    if mirror:
        m = m.flipped(K)
    scales = [0.5, 1.0, 0.8]
    thr, overlap, mc, md = -1.0, 0.4, 300, 40
    d = sd.vl_hog_part_detect(frames, scales, m, CELL, K, thr, overlap=overlap, max_candidates=mc, max_detections=md,
                              multichannel=True, float_frames=True)
    dets, above, parts = dtx._composition(_FloatRoute(sd), frames, scales, m, thr, overlap, mc, md)
    assert np.array_equal(d.above, above)
    rows, prow = dtx._rows(d)
    assert len(rows) > 10
    for i in range(len(frames)):
        sel = d.frame == i
        assert np.array_equal(rows[sel], dets[i]), i
        assert np.array_equal(prow[sel], parts[i]), i
    assert np.any(prow[..., 0] >= 0)


def _integer_frames(seed, n, w, h, quantum=1):
    """8-bit B,G,R frames of planted objects (values multiples of quantum), and boxes."""
    planes, boxes = T.planted_frames(seed, n, w, h, sides=(46, 50))
    rng = np.random.default_rng(seed)
    u8 = []
    for p in planes:
        tint = rng.integers(-30, 31, 3)
        f = np.clip(p.astype(np.int64)[..., None] + tint, 0, 255).astype(np.uint8)
        u8.append(np.ascontiguousarray(f // quantum * quantum))
    return u8, boxes


def test_integer_frames_give_the_8bit_route(sd):
    u8, boxes = _integer_frames(61, 10, 200, 150)
    fl = [f.astype(np.float32) for f in u8]
    rng = np.random.default_rng(5)
    filters = rng.normal(0, 0.2, (2, DD, 4, 5)).astype(np.float32)
    for bil in (False, True):
        kw = dict(bias=[0.1, -0.2], pad=(1, 2), max_detections=40, multichannel=True, bilinear_orientations=bil)
        a = sd.vl_hog_detect(u8, [1.0], filters, CELL, K, -1.0, **kw)
        b = sd.vl_hog_detect(fl, [1.0], filters, CELL, K, -1.0, float_frames=True, **kw)
        assert len(a.frame) > 0
        _same_detections(a, b)
    kw = dict(lam=0.01, rounds=2, negatives_per_frame=16, max_negatives=300, flip_positives=True, multichannel=True)
    a = sd.train_hog_filter(u8, np.arange(10), boxes, [1.0], (SIDE, SIDE), CELL, K, **kw)
    b = sd.train_hog_filter(fl, np.arange(10), boxes, [1.0], (SIDE, SIDE), CELL, K, float_frames=True, **kw)
    assert a.report[0]["positives"] > 0
    assert torch.equal(a.filter.view(torch.int32), b.filter.view(torch.int32)) and np.float32(a.bias) == np.float32(b.bias)
    assert np.array_equal(a.negatives, b.negatives)
    assert [{k: r[k] for k in T.COUNTS + ("solve",)} for r in a.report] == [{k: r[k] for k in T.COUNTS + ("solve",)} for r in b.report]
    # part levels at scale 2: both rules are exact on multiples of 16 at 2x upscales
    q16, _ = _integer_frames(62, 3, 160, 120, quantum=16)
    m = sd.HogPartModel(*dtx._model(np.random.default_rng(8)), max_displacement=None)
    a = sd.vl_hog_part_detect(q16, [1.0], m, CELL, K, -2.0, max_detections=30, multichannel=True)
    b = sd.vl_hog_part_detect([f.astype(np.float32) for f in q16], [1.0], m, CELL, K, -2.0, max_detections=30, multichannel=True,
                              float_frames=True)
    assert len(a.frame) > 0 and np.any(a.placement[..., 0] >= 0)
    _same_detections(a, b)


def _iou(a, b):
    x, y, w, h = (int(v) for v in a)
    bx, by, bw, bh = (int(v) for v in b)
    iw = max(0, min(x + w, bx + bw) - max(x, bx))
    ih = max(0, min(y + h, by + bh) - max(y, by))
    return iw * ih / (w * h + bw * bh - iw * ih)


def test_planted_objects_in_unit_range_frames(sd):
    planes, boxes = T.planted_frames(43, 28, 200, 150, sides=(48, 64))
    frames = _colour(planes, 9)
    assert all(0.0 <= f.min() and f.max() <= 1.25 for f in frames)
    scales = T.detector_scales(200, 150, CELL, SIDE)
    train, test = np.arange(24), np.arange(24, 28)
    hf = sd.train_hog_filter([frames[i] for i in train], np.arange(24), boxes[train], scales, (SIDE, SIDE), CELL, K, lam=0.01,
                             rounds=3, negatives_per_frame=16, max_negatives=4000, flip_positives=True, multichannel=True,
                             float_frames=True)
    held = torch.from_numpy(np.stack([frames[i] for i in test])).cuda()            # a CUDA batch, read in place
    d = sd.vl_hog_detect(held, scales, hf.filter[None], CELL, K, threshold=-10.0, bias=[hf.bias], overlap=0.3, max_detections=4,
                         multichannel=True, float_frames=True)
    for j, i in enumerate(test):
        k = int(np.flatnonzero(d.frame == j)[0])
        iou = _iou(d.boxes[k], boxes[i])
        print(f"held-out frame {i}: top {d.boxes[k].tolist()} score {d.scores[k]:.3f}, object {boxes[i].tolist()}, IoU {iou:.3f}")
        assert iou >= 0.5


def test_python_refusals(sd):
    planes, boxes = T.planted_frames(5, 2, 96, 80, sides=(40, 48))
    fl = _colour(planes, 1)
    u8 = [np.ascontiguousarray((f * 200).astype(np.uint8)) for f in fl]
    filters = np.zeros((1, DD, 4, 4), np.float32)
    m = sd.HogPartModel(*dtx._model(np.random.default_rng(2)), max_displacement=None)
    calls = [lambda fr, **kw: sd.vl_hog_detect(fr, [1.0], filters, CELL, K, 0.0, **kw),
             lambda fr, **kw: sd.train_hog_filter(fr, [0, 1], boxes, [1.0], (4, 4), CELL, K, rounds=0, **kw),
             lambda fr, **kw: sd.vl_hog_part_detect(fr, [1.0], m, CELL, K, 0.0, **kw)]
    for call in calls:
        with pytest.raises(sd.SdError):
            call(fl, multichannel=True)                            # float32 frames need float_frames
        with pytest.raises(ValueError):
            call(fl, float_frames=True)                            # float_frames needs multichannel
        with pytest.raises(ValueError):
            call(u8, multichannel=True, float_frames=True)         # float_frames takes float32 frames only


def test_float_trainer_refusals_write_nothing(sd):
    import ctypes as C
    from superviseddescent_b200 import _capi
    from superviseddescent_b200._capi import HogBoxC, HogImageC, HogImagesC, HogTrainParamC, HogTrainReportC, HogWindowC, ptr
    planes, boxes = T.planted_frames(6, 2, 96, 80, sides=(40, 48))
    f32 = torch.from_numpy(np.stack(_colour(planes, 2))).cuda()
    ctx = sd.default_context()
    hb = (HogBoxC * 2)(*[HogBoxC(i, *(int(v) for v in b)) for i, b in enumerate(boxes)])
    prm = HogTrainParamC(0.01, 0.5, 0.3, 0, 1, 8, 0.5, 50, 20)
    sc = (C.c_double * 1)(1.0)
    filt = torch.full((DD * 4 * 4,), -7.0, device="cuda")
    for data, dtype, p in [(f32, 0, None), (f32, 1, f32.data_ptr() + 2), (f32, 7, None)]:
        ib = HogImagesC()
        ib.d_data, ib.dtype, ib.channels, ib.count = data.data_ptr() if p is None else p, dtype, 3, 2
        ib.frame = HogImageC(96, 80, 0, data.stride(1), data.stride(2), data.stride(3))
        ib.image_stride, ib.d_frames = data.stride(0), None
        bias, nn = C.c_float(-7.0), C.c_int(-1)
        rc = _capi.lib().sd_hog_train_filter_float(ctx.h, C.byref(ib), 0, hb, 2, sc, 1, CELL, K, 1, 4, 4, 0, 0, C.byref(prm), ptr(filt),
                                                   C.byref(bias), (HogTrainReportC * 2)(), (HogWindowC * 50)(), C.byref(nn))
        torch.cuda.synchronize()
        assert rc != 0, (dtype, p)
        assert bool((filt == -7.0).all()) and bias.value == -7.0 and nn.value == -1
